// Weight gradient of the tap-GEMM on the tensor cores (sm_90a, TF32): the training-side twin of tapgemm_tc.cu.
//
//   dW[slab][k][n] += sum over output pixels (b, fo, t) of  A(b, fi, t + dt, k) * dY(b, fo, t, n)
//
// is, per slab, a GEMM whose reduction axis is the pixel axis -- the axis that is NOT contiguous in the channels-last tensors.  Both
// operands are therefore MN-major.  wgmma reads tf32 operands from shared memory K-major only, so this kernel keeps the TMA /
// mbarrier pipeline and feeds mma.sync.m16n8k8 (tf32) from registers: the fragment loads do the transposition.  A TMA box is
// 32 channels x 32 consecutive frames of one (b, f) row, SWIZZLE_128B (row = frame, 128 B of channels, 16-byte unit ^ (frame % 8)):
// no transposition pass, no im2col: the tap shift is the box coordinate, borders and tails are TMA zero fill.
//
//   D (registers) : 128 output channels n (16 per warp) x BN <= 128 input channels k (32-channel boxes taken from the
//                   concatenation of the two source tensors of a skip connection; a box never straddles them)
//   A (smem)      : dY tile  [32 frames][128 n]  = 4 boxes, 16 KB
//   B (smem)      : act tile [32 frames][BN k]   = BN/32 boxes
// One CTA owns one (slab, n-tile, k-tile) and a strided subset of the 32-frame chunks (split-K over pixels); warp 8 = TMA producer,
// warps 0..7 = MMA, then red.global.add.f32 into dW in the parameter's own layout (dW is zeroed by the
// caller; same contract as the SIMT kernel in train.cu).  The tensor core reads fp32 bit patterns and ignores the low 13 mantissa
// bits (truncation, as cuDNN's TF32 convolutions do): this is the precision-1 training mode, not the parity mode.
#include <cuda.h>
#include "common.cuh"
#include "tc_common.cuh"

namespace aero {

constexpr int kWtMmaWarps = 8;
constexpr int kWtThreads = 32 * kWtMmaWarps + 32;
constexpr int kWtMaxBoxes = 4;          // 32-channel boxes per k-tile: 16 accumulators per box and thread
constexpr int kWtMaxStages = 8;
constexpr int kWtChunk = 32;              // frames per pipeline stage (= 4 MMA steps of K = 8)
constexpr int kWtATile = 128 * 128;       // 4 boxes x 4 KB

struct WgradTcShared {
    uint64_t full[kWtMaxStages];
    uint64_t empty[kWtMaxStages];
};

struct WgradTcArgs {
    float* dw;
    aero_tapgemm_params p;
    int64_t dw_sn, dw_sk, dw_ss;
    int tiles_t, n_tiles, k_tiles, nb1, nb, bpt, BN, splits, stages;   // nb1 / nb: 32-channel boxes of source 1 / of both; bpt: boxes per k-tile
    int d_tt, d_fo, d_b;                                               // `splits` chunks ahead, as (frame-chunk, row, batch) carries
};

// Walks the 32-frame chunks split, split + splits, ... of the (b, fo, frame-chunk) space with carries only: the walkers are single
// on the critical path of the pipeline: no division per chunk.
struct WtWalker {
    int b, fo, tt;
    __device__ __forceinline__ void init(const WgradTcArgs& g, int split) {
        tt = split % g.tiles_t;
        const int row = split / g.tiles_t;
        b = row / g.p.F_out;
        fo = row - b * g.p.F_out;
    }
    __device__ __forceinline__ bool done(const WgradTcArgs& g) const { return b >= g.p.B; }
    __device__ __forceinline__ void next(const WgradTcArgs& g) {
        tt += g.d_tt;
        int carry = 0;
        if (tt >= g.tiles_t) { tt -= g.tiles_t; carry = 1; }
        fo += g.d_fo + carry;
        carry = 0;
        if (fo >= g.p.F_out) { fo -= g.p.F_out; carry = 1; }
        b += g.d_b + carry;
    }
    // input row of this slab for the current output row; false when the tap has none
    __device__ __forceinline__ bool input_row(const aero_tapgemm_params& p, int jf, int r, int tapi, int& fi) const {
        if (p.mode == AERO_TAPS_CONV) {
            fi = fo * p.stride_f + jf - p.pad_f;
        } else {
            const int fof = fo + p.f_out_offset;
            const int qf = fof / p.stride_f;
            if (fof - qf * p.stride_f != r) return false;
            fi = qf - tapi;
        }
        return fi >= 0 && fi < p.F_in;
    }
};

// element (frame f, channel ch) of a 32 x 32 SWIZZLE_128B box at shared address `box`
__device__ __forceinline__ uint32_t wt_lds(uint32_t box, int f, int ch) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(box + (uint32_t)(f * 128 + (((ch >> 2) ^ (f & 7)) << 4) + ((ch & 3) << 2))));
    return v;
}

__global__ void __launch_bounds__(kWtThreads, 2)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap mapA1, const __grid_constant__ CUtensorMap mapA2,
                const __grid_constant__ CUtensorMap mapDy, const WgradTcArgs g) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const aero_tapgemm_params& p = g.p;
    const int stage_bytes = kWtATile + (g.BN / 32) * 4096;
    WgradTcShared* sh = reinterpret_cast<WgradTcShared*>(smem + g.stages * stage_bytes);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // work item of this CTA
    const int kt_i = blockIdx.x % g.k_tiles, nt_i = blockIdx.x / g.k_tiles;
    const int slab = blockIdx.y, split = blockIdx.z;
    const int box0 = kt_i * g.bpt;                                // this k-tile: boxes [box0, box0 + nbox) of the concatenated sources
    const int nbox = min(g.bpt, g.nb - box0);
    const int n0 = nt_i * 128;
    int jf = 0, dt = 0, r = 0, tapi = 0;
    if (p.mode == AERO_TAPS_CONV) {
        jf = slab / p.kt;
        dt = (slab - jf * p.kt) * p.dil_t - p.pad_t;
    } else {
        r = slab % p.stride_f;
        tapi = slab / p.stride_f;
    }

    if (threadIdx.x == 0) {
        for (int s = 0; s < g.stages; ++s) { mbar_init(&sh->full[s], 1); mbar_init(&sh->empty[s], kWtMmaWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kWtMmaWarps) {
        // ===================================================== TMA producer
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA1) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&mapDy) : "memory");
            int stage = 0;
            uint32_t phase = 0;
            const uint32_t tx = (uint32_t)(kWtATile + nbox * 4096);
            WtWalker w;
            for (w.init(g, split); !w.done(g); w.next(g)) {
                int fi;
                if (!w.input_row(p, jf, r, tapi, fi)) continue;
                const int t0 = w.tt * kWtChunk;
                mbar_wait(&sh->empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * stage_bytes;
                mbar_expect_tx(&sh->full[stage], tx);
#pragma unroll
                for (int j = 0; j < 4; ++j) tma_load_4d(sa + j * 4096, &mapDy, &sh->full[stage], n0 + 32 * j, t0, w.fo, w.b);
                for (int j = 0; j < nbox; ++j) {
                    const int gb = box0 + j;
                    const bool s2 = gb >= g.nb1;
                    tma_load_4d(sa + kWtATile + j * 4096, s2 ? &mapA2 : &mapA1, &sh->full[stage], 32 * (s2 ? gb - g.nb1 : gb), t0 + dt, fi, w.b);
                }
                if (++stage == g.stages) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // ===================================================== MMA warps: warp w owns output channels n0 + 16 w .. + 15, all boxes
        const int gq = lane >> 2, c = lane & 3;
        float acc[kWtMaxBoxes][4][4];
#pragma unroll
        for (int j = 0; j < kWtMaxBoxes; ++j)
#pragma unroll
            for (int t = 0; t < 4; ++t)
#pragma unroll
                for (int u = 0; u < 4; ++u) acc[j][t][u] = 0.f;
        int stage = 0;
        uint32_t phase = 0;
        int iters = 0;
        WtWalker w;
        for (w.init(g, split); !w.done(g); w.next(g)) {
            int fi_unused;
            if (!w.input_row(p, jf, r, tapi, fi_unused)) continue;         // same enumeration as the producer
            mbar_wait(&sh->full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * stage_bytes);
            const uint32_t abox = sa + (uint32_t)(warp >> 1) * 4096u;
            const int ach = (warp & 1) * 16 + gq;
#pragma unroll
            for (int kk = 0; kk < kWtChunk / 8; ++kk) {
                const int f = 8 * kk + c;
                const uint32_t a0 = wt_lds(abox, f, ach), a1 = wt_lds(abox, f, ach + 8), a2 = wt_lds(abox, f + 4, ach), a3 = wt_lds(abox, f + 4, ach + 8);
#pragma unroll
                for (int j = 0; j < kWtMaxBoxes; ++j) {
                    if (j < nbox) {
                        const uint32_t bbox = sa + kWtATile + (uint32_t)j * 4096u;
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            const uint32_t b0 = wt_lds(bbox, f, 8 * t + gq), b1 = wt_lds(bbox, f + 4, 8 * t + gq);
                            asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                                         : "+f"(acc[j][t][0]), "+f"(acc[j][t][1]), "+f"(acc[j][t][2]), "+f"(acc[j][t][3])
                                         : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&sh->empty[stage]);
            ++iters;
            if (++stage == g.stages) { stage = 0; phase ^= 1; }
        }
        // ===================================================== epilogue: atomics on dW
        if (iters > 0) {
#pragma unroll
            for (int j = 0; j < kWtMaxBoxes; ++j) {
                if (j < nbox) {
                    const int gb = box0 + j;
                    const bool s2 = gb >= g.nb1;
                    const int ch0 = 32 * (s2 ? gb - g.nb1 : gb);
                    const int cnt = min(32, (s2 ? p.C2 : p.C1) - ch0);
                    const int kbase = (s2 ? p.C1 : 0) + ch0;
#pragma unroll
                    for (int t = 0; t < 4; ++t)
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            const int n = n0 + 16 * warp + gq + (u >> 1) * 8, kc = 8 * t + 2 * c + (u & 1);
                            if (n < p.N && kc < cnt)
                                atomicAdd(g.dw + (int64_t)n * g.dw_sn + (int64_t)slab * g.dw_ss + (int64_t)(kbase + kc) * g.dw_sk, acc[j][t][u]);
                        }
                }
            }
        }
    }
}

static int wt_map(CUtensorMap* m, const void* base, int C, int T, int F, int B, int64_t sb, int64_t sf, int64_t st) {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)T, (uint64_t)F, (uint64_t)B};
    int64_t s1 = st, s2 = sf, s3 = sb;
    if (s2 <= 0) s2 = s1 * T;                   // size-1 dimensions: any legal stride
    if (s3 <= 0) s3 = s2 * F;
    uint64_t strides[3] = {(uint64_t)s1 * 4, (uint64_t)s2 * 4, (uint64_t)s3 * 4};
    uint32_t box[4] = {32, (uint32_t)kWtChunk, 1, 1};
    return encode_map(m, base, 4, dims, strides, box, 0, 4);
}

bool wgrad_tc_eligible(const aero_tapgemm_params& p, const void* a1, const void* a2, const void* dy) {
    if (p.mode != AERO_TAPS_CONV && p.mode != AERO_TAPS_CONVT) return false;
    if (p.N < 16 || p.N % 4 || p.C1 % 4 || p.C2 % 4 || p.C1 + p.C2 < 16) return false;
    auto ok = [](int64_t sb, int64_t sf, int64_t st) { return sb % 4 == 0 && sf % 4 == 0 && st % 4 == 0 && st > 0; };
    if (p.C1 && !ok(p.a1_sb, p.a1_sf, p.a1_st)) return false;
    if (p.C2 && !ok(p.a2_sb, p.a2_sf, p.a2_st)) return false;
    if (!ok(p.o_sb, p.o_sf, p.o_st)) return false;
    if (((uintptr_t)a1 | (uintptr_t)a2 | (uintptr_t)dy) & 15) return false;
    return true;
}

int wgrad_tc_launch(const float* a1, const float* a2, const float* dy, float* dw, const aero_tapgemm_params& p, int64_t dw_sn, int64_t dw_sk,
                    int64_t dw_ss, cudaStream_t st) {
    WgradTcArgs g;
    g.dw = dw; g.p = p; g.dw_sn = dw_sn; g.dw_sk = dw_sk; g.dw_ss = dw_ss;
    g.tiles_t = cdiv(p.T, kWtChunk);
    g.n_tiles = cdiv(p.N, 128);
    // B tile = up to kWtMaxBoxes 32-channel boxes taken from the concatenation of the two sources (a box never straddles them)
    g.nb1 = cdiv(p.C1, 32);
    g.nb = g.nb1 + cdiv(p.C2, 32);
    g.k_tiles = cdiv(g.nb, kWtMaxBoxes);
    g.bpt = cdiv(g.nb, g.k_tiles);
    g.BN = 32 * g.bpt;
    CUtensorMap mA1, mA2, mDy;
    int rc;
    if (p.C1 && (rc = wt_map(&mA1, a1, p.C1, p.T_in, p.F_in, p.B, p.a1_sb, p.a1_sf, p.a1_st)) != AERO_OK) return rc;
    if (p.C2 && (rc = wt_map(&mA2, a2, p.C2, p.T_in, p.F_in, p.B, p.a2_sb, p.a2_sf, p.a2_st)) != AERO_OK) return rc;
    if (!p.C1) mA1 = mA2;
    if (!p.C2) mA2 = mA1;
    if ((rc = wt_map(&mDy, dy, p.N, p.T, p.F_out, p.B, p.o_sb, p.o_sf, p.o_st)) != AERO_OK) return rc;
    const int stage_bytes = kWtATile + (g.BN / 32) * 4096;
    const int fixed = (int)sizeof(WgradTcShared) + 1024;
    g.stages = 3;                                 // ~97 KB with barriers and alignment: two CTAs per SM, one's fragment loads overlap the other's MMAs
    const size_t smem = (size_t)g.stages * stage_bytes + fixed;
    const int nslab = (p.mode == AERO_TAPS_CONVT) ? p.kf : p.kf * p.kt;
    const int64_t n_chunks = (int64_t)p.B * p.F_out * g.tiles_t;
    const int64_t items = (int64_t)g.k_tiles * g.n_tiles * nslab;
    static int num_sms = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    // split the pixel axis: two CTAs per SM are resident (the pipeline takes the shared memory), so the grid should be a whole number of
    // waves.  Among the split counts that give 2 .. 6 waves pick the one with the fullest last wave; a split keeps at least 8 chunks so
    // that the atomics stay a small fraction of the work.
    const int64_t max_splits = n_chunks / 8 > 0 ? n_chunks / 8 : 1;
    const int64_t slots = (int64_t)2 * num_sms;
    int64_t lo = cdiv(2 * slots, items), hi = cdiv(6 * slots, items);
    if (lo > max_splits) lo = max_splits;
    if (hi > max_splits) hi = max_splits;
    if (hi > 65535) hi = 65535;
    if (lo < 1) lo = 1;
    if (hi < lo) hi = lo;
    int64_t splits = lo;
    double best_eff = 0.0;
    for (int64_t sp = lo; sp <= hi; ++sp) {
        const int64_t ctas = items * sp;
        const double eff = (double)ctas / (double)(cdiv(ctas, slots) * slots);
        if (eff > best_eff + 0.02) { best_eff = eff; splits = sp; }      // prefer fewer splits unless clearly fuller
    }
    g.splits = (int)splits;
    g.d_tt = g.splits % g.tiles_t;
    const int d_row = g.splits / g.tiles_t;
    g.d_fo = d_row % p.F_out;
    g.d_b = d_row / p.F_out;
    if (nslab > 65535 || items / nslab > 2147483647LL) { set_error("aero_tapgemm_wgrad(tensor cores): grid too large"); return AERO_ERR_INVALID; }
    cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    dim3 grid((unsigned)(items / nslab), (unsigned)nslab, (unsigned)splits);
    wgrad_tc_kernel<<<grid, kWtThreads, smem, st>>>(mA1, mA2, mDy, g);
    return check_launch("aero_tapgemm_wgrad(tensor cores)");
}

}  // namespace aero
