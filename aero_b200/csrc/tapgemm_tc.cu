// Host side of the tensor-core tap-GEMM: TMA descriptors, tile-width choice, launch.  The kernel is in tapgemm_tc_kernel.cuh.
#include <cuda.h>
#include <mutex>
#include <unordered_map>
#include <string>
#include <cstring>
#include <cstdlib>

#include "tapgemm.cuh"
#include "tc_common.cuh"

namespace aero {

KernelFn tapgemm_tc_kernels_bn32(bool f16a, bool f16o, int amode, bool res, bool stats);
KernelFn tapgemm_tc_kernels_bn64(bool f16a, bool f16o, int amode, bool res, bool stats);
KernelFn tapgemm_tc_kernels_bn96(bool f16a, bool f16o, int amode, bool res, bool stats);
KernelFn tapgemm_tc_kernels_bn128(bool f16a, bool f16o, int amode, bool res, bool stats);
KernelFn tapgemm_tc_kernels_bn192(bool f16a, bool f16o, int amode, bool res, bool stats);
KernelFn tapgemm_tc_kernels_bn256(bool f16a, bool f16o, int amode, bool res, bool stats);

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

struct MapKey {
    const void* base;
    uint64_t d[4], s[3];
    uint32_t box[4], rank, swz, pad_;
    bool operator==(const MapKey& o) const { return std::memcmp(this, &o, sizeof(MapKey)) == 0; }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
        size_t h = 1469598103934665603ull;
        for (size_t i = 0; i < sizeof(MapKey) / 8; ++i) h = (h ^ w[i]) * 1099511628211ull;
        return h;
    }
};

int encode_map(CUtensorMap* out, const void* base, uint32_t rank, const uint64_t* dims, const uint64_t* strides_bytes,
               const uint32_t* box, int swizzle_mode, int elem_bytes) {
    static std::mutex mu;
    static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
    MapKey key;
    std::memset(&key, 0, sizeof(key));
    key.base = base;
    key.rank = rank;
    key.swz = (uint32_t)swizzle_mode | ((uint32_t)elem_bytes << 8);
    for (uint32_t i = 0; i < rank; ++i) { key.d[i] = dims[i]; key.box[i] = box[i]; }
    for (uint32_t i = 0; i + 1 < rank; ++i) key.s[i] = strides_bytes[i];
    {
        std::lock_guard<std::mutex> lk(mu);
        auto it = cache.find(key);
        if (it != cache.end()) { *out = it->second; return AERO_OK; }
    }
    EncodeTiledFn enc = get_encode();
    if (!enc) { set_error("cuTensorMapEncodeTiled not available from the driver"); return AERO_ERR_UNSUPPORTED; }
    cuuint64_t gd[4];
    cuuint64_t gs[3];
    cuuint32_t bx[4], es[4];
    for (uint32_t i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
    for (uint32_t i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
    CUresult r = enc(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<void*>(base), gd, gs, bx, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle_mode == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): rank %u dims %llu %llu %llu %llu", (int)r, rank,
                  (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0),
                  (unsigned long long)(rank > 3 ? dims[3] : 0));
        return AERO_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(mu);
    if (cache.size() > 4096) cache.clear();
    cache.emplace(key, *out);
    return AERO_OK;
}

// Shared memory of a CTA besides the pipeline stages: barriers / scratch, the bias of every column (padded to whole tiles) and the
// accumulator staging tile (the wide widths stage kSliceBN columns at a time).
static int tc_fixed_smem(int N, int BN) {
    return (int)sizeof(TcShared) + cdiv(N, BN) * BN * 4 + kBM * ((BN > kMaxBN ? kSliceBN : BN) + 4) * 4 + 1024;
}
// Pipeline depth: the producer runs ahead across tiles, so depth is set by bytes in flight, not by the K length: as many stages as
// fit.  Fewer than two cannot run (a stage is released only after the next one's wgmmas are issued).
static int tc_stages(int N, int BN) {
    if (N > (1 << 20)) return 0;
    const int st = (227 * 1024 - tc_fixed_smem(N, BN)) / (kATileBytes + BN * 128);
    return st > kMaxStages ? kMaxStages : st;
}

// Shortest K loop, (C1 + C2) x taps, that takes a wide tile.  A 128 x 256 tile halves the weight bytes each pixel tile pulls
// and cuts the L2 -> SM bytes per FLOP by a quarter, which pays on the tensor-bound convolutions (the shortest of the
// aero_4-16_512_64 forward is encoder.2.conv: 96 x 8 = 768).  The short-K launches (1x1 rewrites, LSTM gate inputs: K x taps
// <= 384 there) are bound by HBM and by the epilogue; a wider tile only coarsens their waves, so they keep the narrow widths.
constexpr int kWideMinKTaps = 512;

// Tile width.  Narrow (32, 64, 96, 128): the narrowest that covers N in the fewest n-tiles of at most 128.  Wide (192, 256):
// FP16 operands, N >= 192 and a K loop of at least kWideMinKTaps, when three pipeline stages and the statistics slots of a
// tile still fit; otherwise the narrow width.
static int pick_bn(const aero_tapgemm_params& p) {
    const int nt = cdiv(p.N, kMaxBN);
    const int narrow = (cdiv(p.N, nt) + 31) & ~31;
    if (p.precision != 2 || p.mode == AERO_TAPS_MIX || p.N < 192) return narrow;
    const int taps = (p.mode == AERO_TAPS_CONV) ? p.kf * p.kt : p.kf / p.stride_f;
    if ((int64_t)(p.C1 + p.C2) * taps < kWideMinKTaps) return narrow;
    const int bn = cdiv(p.N, cdiv(p.N, kWideBN)) <= 192 ? 192 : 256;
    if (tc_stages(p.N, bn) < 3) return narrow;
    if (p.stats_mode == 1) {
        const int Nout = p.glu ? p.N / 2 : p.N;
        if (p.groups < 1 || Nout % p.groups || (p.glu ? bn / 2 : bn) / (Nout / p.groups) + 2 > 8) return narrow;
    }
    return bn;
}

// precision 1: fp32 sources (tf32 wgmma); precision 2: FP16 sources (f16 wgmma).  TMA needs 16-byte global strides:
// channel counts / strides in multiples of 4 fp32 or 8 halves.
bool tapgemm_tc_eligible(const aero_tapgemm_params& p) {
    const bool f16 = (p.flags & AERO_TG_A_F16) != 0;
    const int q = f16 ? 8 : 4;
    if (p.mode == AERO_TAPS_MIX)
        return p.w_sb == 0 && p.C1 % q == 0 && p.C2 == 0 && p.a1_st % q == 0 && p.a1_sb % q == 0 && p.N >= 8 &&
               p.stats_mode == 0 && !p.glu && p.F_out == 1 && p.F_in == 1 && tc_stages(p.N, pick_bn(p)) >= 2;
    if (p.w_sb != 0) return false;                                   // activations-as-weights (FTB frequency mix)
    if (p.act == AERO_ACT_TANH) return false;                        // tanh is built for the SIMT kernels only (SEANet's thin layers)
    if (p.act == AERO_ACT_LEAKY && (p.stats_mode != 0 || p.r_sb != 0 || p.r_sf != 0 || p.r_st != 0))
        return false;                                                // LeakyReLU: plain epilogue only (no residual, no statistics)
    if (tc_stages(p.N, pick_bn(p)) < 2) return false;                // the bias of that many columns leaves no room for a pipeline
    if (p.N < 8) return false;                                       // thin outputs stay on the SIMT path
    const int K = p.C1 + p.C2;
    if (K < 8 || (p.C1 % q) || (p.C2 % q)) return false;
    auto ok_strides = [q](int64_t sb, int64_t sf, int64_t st) { return sb % q == 0 && sf % q == 0 && st % q == 0 && st > 0; };
    if (p.C1 && !ok_strides(p.a1_sb, p.a1_sf, p.a1_st)) return false;
    if (p.C2 && !ok_strides(p.a2_sb, p.a2_sf, p.a2_st)) return false;
    if (p.stats_mode == 1) {
        const int Nout = p.glu ? p.N / 2 : p.N;
        if (p.groups < 1 || Nout % p.groups) return false;
        const int gw = Nout / p.groups;
        const int bn = pick_bn(p);
        if (gw % 8 || (p.glu ? bn / 2 : bn) / gw + 2 > 8) return false;
    }
    return true;
}

static int make_a_map(CUtensorMap* m, const void* base, int C, const aero_tapgemm_params& p, int64_t sb, int64_t sf, int64_t st, int esz) {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)p.T_in, (uint64_t)p.F_in, (uint64_t)p.B};
    int64_t s1 = st, s2 = sf, s3 = sb;
    if (s2 <= 0) s2 = s1 * p.T_in;              // size-1 dimensions: any legal stride
    if (s3 <= 0) s3 = s2 * p.F_in;
    uint64_t strides[3] = {(uint64_t)s1 * esz, (uint64_t)s2 * esz, (uint64_t)s3 * esz};
    uint32_t box[4] = {(uint32_t)(128 / esz), (uint32_t)kBM, 1, 1};
    return encode_map(m, base, 4, dims, strides, box, 0, esz);
}

// tuning knobs (tools/kprof.py), read from the environment ONCE when the library first launches this kernel: the launch
// path itself never calls getenv.  -1 = not set.
struct TcKnobs {
    int direct_f32 = -1, direct_f16 = -1, stages = -1;
    TcKnobs() {
        auto rd = [](const char* name, int& v) { if (const char* e = getenv(name)) v = atoi(e); };
        rd("AERO_TC_DIRECT_F32", direct_f32); rd("AERO_TC_DIRECT_F16", direct_f16); rd("AERO_TC_STAGES", stages);
    }
};
static const TcKnobs& knobs() { static const TcKnobs k; return k; }

int tapgemm_tc_launch(const TapGemmArgs& g0, cudaStream_t st) {
    const TcKnobs& kn = knobs();
    TapGemmArgs g = g0;
    const aero_tapgemm_params& p = g.p;
    const bool f16a = p.precision == 2, f16o = (p.flags & AERO_TG_OUT_F16) != 0;
    const int esz = f16a ? 2 : 4, kBKc = 128 / esz;
    const int K = p.C1 + p.C2;
    const int BN = pick_bn(p);
    const int nslab = (p.mode == AERO_TAPS_CONVT) ? p.kf : p.kf * p.kt;
    CUtensorMap mA1, mA2, mW;
    int rc;
    const bool mix = p.mode == AERO_TAPS_MIX;
    if (mix) {
        // activations as [K = C1 rows][M = T contiguous] per batch item
        uint64_t dims[3] = {(uint64_t)p.T, (uint64_t)p.C1, (uint64_t)p.B};
        uint64_t strides[2] = {(uint64_t)p.a1_st * esz, (uint64_t)(p.a1_sb > 0 ? p.a1_sb : (int64_t)p.a1_st * p.C1) * esz};
        uint32_t box[3] = {(uint32_t)(f16a ? 64 : 32), (uint32_t)kBKc, 1};
        if ((rc = encode_map(&mA1, g.a1, 3, dims, strides, box, 0, esz)) != AERO_OK) return rc;
    } else if (p.C1) { if ((rc = make_a_map(&mA1, g.a1, p.C1, p, p.a1_sb, p.a1_sf, p.a1_st, esz)) != AERO_OK) return rc; }
    if (p.C2) { if ((rc = make_a_map(&mA2, g.a2, p.C2, p, p.a2_sb, p.a2_sf, p.a2_st, esz)) != AERO_OK) return rc; }
    if (!p.C1) mA1 = mA2;
    if (!p.C2) mA2 = mA1;
    {
        // weights are stored K-major W[slab][pad4(N)][Kp], Kp = K (fp32) or K rounded up to 8 (FP16: 16-byte rows)
        const uint64_t npad = (uint64_t)((p.N + 3) & ~3);
        const uint64_t kp = f16a ? (uint64_t)((K + 7) & ~7) : (uint64_t)K;
        uint64_t dims[3] = {(uint64_t)K, npad, (uint64_t)nslab};
        uint64_t strides[2] = {kp * esz, kp * npad * esz};
        uint32_t box[3] = {(uint32_t)kBKc, (uint32_t)BN, 1};
        if ((rc = encode_map(&mW, g.w, 3, dims, strides, box, 0, esz)) != AERO_OK) return rc;
    }
    g.tiles_t = cdiv(p.T, kBM);
    g.direct_f32 = 0;
    g.direct_f16 = 2;       // GLU outputs take the direct form (one 16-byte store per lane), the others the transpose
    if (kn.direct_f32 >= 0) g.direct_f32 = kn.direct_f32;
    if (kn.direct_f16 >= 0) g.direct_f16 = kn.direct_f16;
    const int64_t tiles = (int64_t)p.B * p.F_out * g.tiles_t;
    if (tiles > 2147483647LL) { set_error("aero_tapgemm_fwd: too many tiles"); return AERO_ERR_INVALID; }
    {
        const uint32_t divs[3] = {(uint32_t)cdiv(p.N, BN), (uint32_t)g.tiles_t, (uint32_t)p.F_out};
        for (int i = 0; i < 3; ++i) {
            uint32_t s = 0;
            while ((1ull << s) < divs[i]) ++s;                         // ceil(log2 d)
            const uint64_t two = 1ull << (31 + s);
            g.dv_mul[i] = (uint32_t)((two + divs[i] - 1) / divs[i]);   // ceil(2^(31+s) / d) <= 2^32 - 1 (d = 1: 2^31)
            g.dv_shr[i] = 31 + s;
        }
    }
    const int stage_bytes = kATileBytes + BN * 128;
    const int fixed = tc_fixed_smem(p.N, BN);
    int kStages = tc_stages(p.N, BN);
    if (kStages < 2) {
        set_error("aero_tapgemm_fwd(wgmma): N = %d leaves no shared memory for the pipeline", p.N);
        return AERO_ERR_UNSUPPORTED;
    }
    if (kn.stages >= 2 && kn.stages < kStages) kStages = kn.stages;
    const size_t smem = (size_t)kStages * stage_bytes + fixed;
    // epilogue template mode: 0-2 = act, 3 = GLU, 4 = AERO_ACT_LEAKY (the engine never combines GLU with an activation)
    const int amode = p.glu ? 3 : (p.act == AERO_ACT_LEAKY ? 4 : p.act);
    if (p.glu && p.act != AERO_ACT_NONE) { set_error("aero_tapgemm_fwd(wgmma): GLU with an activation is not supported"); return AERO_ERR_UNSUPPORTED; }
    const bool res = g.residual != nullptr, stats = p.stats_mode != 0;
    const KernelFn kern = BN == 32 ? tapgemm_tc_kernels_bn32(f16a, f16o, amode, res, stats)
                        : BN == 64 ? tapgemm_tc_kernels_bn64(f16a, f16o, amode, res, stats)
                        : BN == 96 ? tapgemm_tc_kernels_bn96(f16a, f16o, amode, res, stats)
                        : BN == 128 ? tapgemm_tc_kernels_bn128(f16a, f16o, amode, res, stats)
                        : BN == 192 ? tapgemm_tc_kernels_bn192(f16a, f16o, amode, res, stats)
                                    : tapgemm_tc_kernels_bn256(f16a, f16o, amode, res, stats);
    if (!kern) {
        set_error("aero_tapgemm_fwd(wgmma): epilogue (act %d, residual %d, stats %d) is not built for operands %s / outputs %s",
                  amode, (int)res, (int)stats, f16a ? "f16" : "tf32", f16o ? "f16" : "f32");
        return AERO_ERR_UNSUPPORTED;
    }
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    // persistent grid: one CTA per SM (the pipeline and the staging tile take the shared memory), never more than tiles
    static int num_sms = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    const int n_tiles = cdiv(p.N, BN);
    const int64_t tiles_total = tiles * n_tiles;
    if (tiles_total > 2147483647LL) { set_error("aero_tapgemm_fwd: too many tiles"); return AERO_ERR_INVALID; }
    const int64_t want = num_sms;
    g.last_tile = (int)tiles_total - 1;
    dim3 grid((unsigned)(tiles_total < want ? tiles_total : want));
    kern<<<grid, kThreads, smem, st>>>(mA1, mA2, mW, g, kStages, n_tiles, (int)tiles_total);
    return check_launch("aero_tapgemm_fwd(wgmma)");
}

}  // namespace aero
