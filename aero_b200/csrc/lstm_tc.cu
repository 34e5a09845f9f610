// Persistent BiLSTM recurrence on the Hopper tensor cores (wgmma, sm_90a).  See include/aero_b200.h (aero_lstm_rec_fwd,
// precision = 1).
//
// Per step the recurrent term is the small GEMM  D[4H gate rows x sequences] = W_hh[4H x H] * h^T[H x sequences]:
//   A = W_hh, FP16, held in REGISTERS as the wgmma A fragment for the whole sequence.  The 4H gate rows are packed densely in
//       PyTorch's order, dense row R = gate * H + cell, into KS = ceil(4H / 64) = ceil(H / 16) m64 tiles; K = H runs in KS
//       k16 steps (zero beyond H).  Tile t, k-step k is 4 registers per thread; one MMA warpgroup holds all tiles when
//       KS <= 4 (H <= 64: 4 x 4 x 4 = 64 registers, 36 at H = 48), two warpgroups split them when KS <= 6 (H <= 96: 3 x 6 x 4 = 72
//       each).  They are gathered once per CTA from the re-ordered rows lstm_gate_reorder / lstm_whh_fp16 produce (L2-resident,
//       4-byte loads), so no shared-memory traffic for A remains in the step;
//   B = h of the previous step, FP16, written by the cell-update threads straight into the swizzled (SWIZZLE_128B, K-major)
//       shared-memory operand layout, one NT x 64-column tile per 64 cells (NT = wgmma N = 8 or 16 sequences);
//   D = KS tiles of 64 x NT fp32 (accumulated in fp32; only the order of the K sum differs from a plain dot product), staged
//       transposed in shared memory, sAcc[sequence][R] with a row stride of 64 KS + 4 floats: the MMA threads' scalar stores and
//       the cell threads' float2 reads of two adjacent cells of one gate are both free of bank conflicts.
// Two sequence groups per CTA (ping-pong): the MMA warpgroup(s) serve group 0 and group 1 alternately, so one group's wgmmas run
// while the other group's cell warps do their exp-heavy update.  Each group has its own h_ready / acc_ready mbarrier pair, B
// operand and staging buffer, and four cell-update warps.  A cell thread owns up to kItems (sequence, cell pair) items of its
// group, two adjacent cells each, and only live cells (< H) are computed: gate pre-activations load as float2 / half2 (the
// input projection keeps PyTorch's [dir][i,f,g,o][H] column order) and are requested into registers a whole step ahead and into
// L2 two steps ahead; c stays in registers.
#include <cuda_fp16.h>
#include <algorithm>
#include "tc_common.cuh"

#ifdef AERO_TC_TRACE
__device__ long long g_lstm_trace[128 * 8];
#define LSTM_TRACE(slot, step) do { if (blockIdx.x == 0 && blockIdx.y == 0 && (step) < 128) g_lstm_trace[(step) * 8 + (slot)] = clock64(); } while (0)
extern "C" int aero_debug_lstm_trace(long long* host) {
    return cudaMemcpyFromSymbol(host, g_lstm_trace, sizeof(g_lstm_trace)) == cudaSuccess ? 0 : -1;
}
#else
#define LSTM_TRACE(slot, step) do { } while (0)
#endif

namespace aero {

constexpr int kCellThreads = 128;   // cell-update threads per sequence group
constexpr int kItems = 3;           // cell pairs per cell thread (all of one sequence)

struct LstmTcShape {
    int S, nt, ctas_per_dir, tps;       // sequences per group, wgmma N, CTAs per direction, cell threads per sequence
};

struct LstmTcShared {
    uint64_t acc_ready[2];
    uint64_t h_ready[2];
};

// ex2.approx / rcp.approx: <= 2 ulp each, i.e. ~1e-7 relative on the gates (far below the operand rounding)
__device__ __forceinline__ float fast_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float fast_rcp(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float2 ld2f(const float* p) { return *reinterpret_cast<const float2*>(p); }
__device__ __forceinline__ float2 to_f2(float2 v) { return v; }
__device__ __forceinline__ float2 to_f2(__half2 v) { return __half22float2(v); }
template <typename TG> struct Pair;
template <> struct Pair<float> { using T = float2; };
template <> struct Pair<__half> { using T = __half2; };
__device__ __forceinline__ void st2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
__device__ __forceinline__ void st2(__half* p, float a, float b) { *reinterpret_cast<uint32_t*>(p) = pack_half2_sat(a, b); }

// KS = ceil(H / 16): m64 tiles of gate rows == k16 steps of K.  NT: wgmma N (8 or 16 sequences per group).
template <int KS> struct LstmTcCfg {
    static constexpr int kWG = KS > 4 ? 2 : 1;                  // MMA warpgroups
    static constexpr int kTW = (KS + kWG - 1) / kWG;            // m64 tiles per MMA warpgroup (KS = 5: the last one is zero)
    static constexpr int kLdr = 64 * kWG * kTW + 4;             // staged accumulator row stride (floats), == 4 mod 32
    static constexpr int kThreads = 128 * kWG + 2 * kCellThreads;
};

template <int KS, int NT, typename TO, typename TG>
__global__ void __launch_bounds__(LstmTcCfg<KS>::kThreads, 1)
lstm_tc_kernel(const __half* __restrict__ whh, const TG* __restrict__ gin, const float* __restrict__ bias_pad,
               TO* __restrict__ hout, const aero_lstm_params p, const int S, const int tps) {
    using Cfg = LstmTcCfg<KS>;
    constexpr int kTW = Cfg::kTW, kLdr = Cfg::kLdr, NWG = Cfg::kWG;
    constexpr int nK = (KS + 3) / 4;                    // 64-column B chunks
    constexpr int kBTile = NT * 128;                    // bytes of one 64-column B chunk (NT rows of 128 B)
    using TG2 = typename Pair<TG>::T;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int H = p.H;
    uint8_t* sB = smem;                                 // [2][nK][kBTile]
    float* sAcc = reinterpret_cast<float*>(sB + 2 * nK * kBTile);   // [2][NT][kLdr]
    LstmTcShared* sh = reinterpret_cast<LstmTcShared*>(sAcc + 2 * NT * kLdr);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.y;
    const int n_seq = p.rows * p.n_win;
    // group g of this CTA: sequences [seq0 + g * S, + live[g]); group 0 is never empty, group 1 may be
    const int seq0 = blockIdx.x * 2 * S;
    const int live0 = min(S, n_seq - seq0), live1 = max(0, min(S, n_seq - seq0 - S));

    if (threadIdx.x == 0) {
        for (int g = 0; g < 2; ++g) {
            mbar_init(&sh->acc_ready[g], 128 * NWG);
            mbar_init(&sh->h_ready[g], max(1, (g ? live1 : live0) * tps));   // the cell threads that own a sequence
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < 2 * nK * kBTile / 4; i += blockDim.x) reinterpret_cast<float*>(sB)[i] = 0.f;
    fence_proxy_async_smem();
    __syncthreads();

    if (warp < 4 * NWG) {
        // ===================================================== MMA warpgroup(s)
        const int wg = warp >> 2, wl = warp & 3;
        // A fragment of m64k16 (FP16): reg r of lane l holds rows 16 wl + l/4 (+8 if r odd), columns 2 (l%4) (+8 if r >= 2), +1.
        // Dense row R = gate * H + cell comes from the re-ordered row of lstm_gate_reorder (GPT = 1 if H > 64 else 2).
        const int kp = 64 * nK;                         // fp16 per re-ordered row
        const int nM = H > 64 ? 4 : 2;
        uint32_t a[kTW][KS][4];
#pragma unroll
        for (int lt = 0; lt < kTW; ++lt)
#pragma unroll
            for (int k = 0; k < KS; ++k)
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int R = (wg * kTW + lt) * 64 + wl * 16 + (lane >> 2) + 8 * (r & 1);
                    const int col = 16 * k + 2 * (lane & 3) + 8 * (r >> 1);
                    uint32_t v = 0u;
                    if (R < 4 * H && col < H) {
                        const int gate = R / H, cell = R - gate * H;
                        const int src = H > 64 ? gate * 128 + cell
                                               : (gate >> 1) * 128 + (cell >> 4) * 32 + (gate & 1) * 16 + (cell & 15);
                        v = __ldg(reinterpret_cast<const uint32_t*>(whh + (size_t)(dir * nM * 128 + src) * kp + col));
                    }
                    a[lt][k][r] = v;
                }
        // B descriptors: group g, k-step k -> chunk k / 4, +32 bytes per k16 inside the 128-byte swizzled row
        const uint64_t db0 = make_desc_kmajor<128>(smem_u32(sB));
        const int ng = live1 > 0 ? 2 : 1;
        float* const arow = sAcc + 2 * (lane & 3) * kLdr + wg * kTW * 64 + wl * 16 + (lane >> 2);
        for (int s = 1; s < p.steps; ++s) {
            for (int g = 0; g < ng; ++g) {
                mbar_wait(&sh->h_ready[g], (uint32_t)((s - 1) & 1));
                if (g == 0) LSTM_TRACE(0, s);
                const uint64_t db = db0 + (uint64_t)(g * ((nK * kBTile) >> 4));
                float d[kTW][NT / 2];      // first written by the first wgmma of each chain (scale-d = 0)
                wgmma_fence();
#pragma unroll
                for (int lt = 0; lt < kTW; ++lt)
#pragma unroll
                    for (int k = 0; k < KS; ++k)
                        Wgmma<NT, true, 0>::rs(d[lt], a[lt][k], db + (uint64_t)((k >> 2) * (kBTile >> 4) + 2 * (k & 3)), k == 0 ? 0u : 1u);
                wgmma_commit();
                wgmma_wait<0>();
                float* const acc = arow + g * NT * kLdr;
#pragma unroll
                for (int lt = 0; lt < kTW; ++lt)
#pragma unroll
                    for (int j = 0; j < NT / 8; ++j)
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            acc[(8 * j + (e & 1)) * kLdr + lt * 64 + 8 * (e >> 1)] = d[lt][4 * j + e];
                mbar_arrive(&sh->acc_ready[g]);
                if (g == 0) LSTM_TRACE(1, s);
            }
        }
    } else {
        // ===================================================== cell update: four warps per group
        const int g = (warp - 4 * NWG) >> 2;
        const int t = threadIdx.x - 128 * NWG - g * kCellThreads;
        // thread t: local sequence n = t / tps, cell pairs pp + tps j (j < kItems, pair < H / 2): cells 2 pair, 2 pair + 1
        const int n = t / tps, pp = t - n * tps;
        if (n >= (g ? live1 : live0)) return;
        const int hp = H >> 1;
        const int half = p.win_stride / 2;
        const int dpos = dir ? -1 : 1;
        const int pos0 = dir ? p.steps - 1 : 0;
        const int ldg = 8 * H;                          // gin row: [dir][i,f,g,o][H], PyTorch's own order

        // A step s reads the input projection iff (unsigned)(s - g_lo) < g_len (else the frame is zero padding: bias only)
        // and writes its output iff (unsigned)(s - w_lo) < w_len (window crop of modules.py:53-59 and the T limit).
        const int sq = seq0 + g * S + n;
        const int row = sq / p.n_win, k = sq - row * p.n_win;
        const int f0 = k * p.win_stride;                                  // first frame of the window
        const int cell0 = 2 * pp, cstep = 2 * tps;                        // cells of item j: cell0 + cstep j, +1
        const int gcol = dir * 4 * H + cell0;
        int goff = (p.in_windowed ? (sq * p.steps + pos0) : (row * p.T + f0 + pos0)) * ldg + gcol;
        // valid input positions of this window: frames < T.  position -> step: dir 0: s = pos; dir 1: s = steps-1-pos
        const int in_hi = p.in_windowed ? p.steps : max(0, min(p.steps, p.T - f0));
        const int g_lo = dir ? p.steps - in_hi : 0, g_len = in_hi;
        int ooff = (p.out_windowed ? (sq * p.steps + pos0) : (row * p.T + f0 + pos0)) * 2 * H + dir * H + cell0;
        // kept output positions [lo, hi) (window crop of modules.py:53-59) intersected with frames < T
        int lo = 0, hi = p.steps;
        if (!p.out_windowed) {
            lo = (k == 0) ? 0 : half;
            hi = min((k == p.n_win - 1) ? p.steps : p.steps - half, p.T - f0);
        }
        const int w_lo = dir ? p.steps - hi : lo, w_len = max(0, hi - lo);
        const float* const accn = sAcc + (g * NT + n) * kLdr + cell0;
        bool ok[kItems];
        uint32_t baddr[kItems];
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
            ok[j] = pp + tps * j < hp;
            // swizzled B-operand address of (sequence n, k = cell), fp16: chunk cell / 64, row n (128 B), 16-byte unit
            // (cell % 64) / 8 XOR-ed with n % 8, then (cell % 8) * 2 bytes
            const int cell = cell0 + cstep * j;
            baddr[j] = smem_u32(sB) + (uint32_t)((g * nK + (cell >> 6)) * kBTile + (n >> 3) * 1024 + (n & 7) * 128 +
                                                 ((((cell & 63) >> 3) ^ (n & 7)) << 4) + ((cell & 7) << 1));
        }
        const int gstep = dpos * ldg, ostep = dpos * 2 * H;

        float c_state[kItems][2];
        TG2 gn[kItems][4];      // next step's gate pre-activations, kept in the storage type until the step that uses them
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
            c_state[j][0] = c_state[j][1] = 0.f;
            if (ok[j] && (unsigned)(0 - g_lo) < (unsigned)g_len) {
#pragma unroll
                for (int q = 0; q < 4; ++q) gn[j][q] = *reinterpret_cast<const TG2*>(gin + goff + cstep * j + q * H);
            }
        }
        goff += gstep;
        for (int s = 0; s < p.steps; ++s) {
            float2 gi[kItems][4];
            const bool real = (unsigned)(s - g_lo) < (unsigned)g_len;
            const bool real_next = s + 1 < p.steps && (unsigned)(s + 1 - g_lo) < (unsigned)g_len;
            const bool real_next2 = s + 2 < p.steps && (unsigned)(s + 2 - g_lo) < (unsigned)g_len;
#pragma unroll
            for (int j = 0; j < kItems; ++j) {
                if (!ok[j]) continue;
#pragma unroll
                for (int q = 0; q < 4; ++q) gi[j][q] = real ? to_f2(gn[j][q]) : ld2f(bias_pad + gcol + cstep * j + q * H);
                if (real_next) {
#pragma unroll
                    for (int q = 0; q < 4; ++q) gn[j][q] = *reinterpret_cast<const TG2*>(gin + goff + cstep * j + q * H);
                }
                // and the step after that into L2: a register load a single step ahead does not cover HBM latency under load
                if (real_next2) {
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        asm volatile("prefetch.global.L2 [%0];" ::"l"(gin + goff + gstep + cstep * j + q * H));
                }
            }
            goff += gstep;
            if (g == 0 && t == 0) LSTM_TRACE(2, s);
            if (s > 0) mbar_wait(&sh->acc_ready[g], (uint32_t)((s - 1) & 1));
            if (g == 0 && t == 0) LSTM_TRACE(3, s);
            const bool store = (unsigned)(s - w_lo) < (unsigned)w_len;
#pragma unroll
            for (int j = 0; j < kItems; ++j) {
                if (!ok[j]) continue;
                float act[4][2];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float2 acc = s > 0 ? *reinterpret_cast<const float2*>(accn + cstep * j + q * H) : make_float2(0.f, 0.f);
                    // PyTorch gate order 0 i, 1 f, 2 g, 3 o; gate 2 is tanh = 2*sigmoid(2x) - 1: fold into scale / affine
                    const float k_in = (q == 2) ? -2.885390081777927f : -1.4426950408889634f;   // -(1|2) * log2(e)
                    const float k_mul = (q == 2) ? 2.0f : 1.0f, k_add = (q == 2) ? -1.0f : 0.0f;
                    act[q][0] = fmaf(k_mul, fast_rcp(1.0f + fast_ex2(k_in * (acc.x + gi[j][q].x))), k_add);
                    act[q][1] = fmaf(k_mul, fast_rcp(1.0f + fast_ex2(k_in * (acc.y + gi[j][q].y))), k_add);
                }
                float h[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float c = fmaf(act[1][e], c_state[j][e], act[0][e] * act[2][e]);
                    c_state[j][e] = c;
                    const float th = fmaf(2.0f, fast_rcp(1.0f + fast_ex2(-2.885390081777927f * c)), -1.0f);
                    h[e] = round_tf32_rna(act[3][e] * th);
                }
                const __half2 hh = __floats2half2_rn(h[0], h[1]);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(baddr[j]), "r"(*reinterpret_cast<const uint32_t*>(&hh)) : "memory");
                if (store) st2(hout + ooff + cstep * j, h[0], h[1]);
            }
            ooff += ostep;
            if (g == 0 && t == 0) LSTM_TRACE(5, s);
            if (s + 1 < p.steps) {
                fence_proxy_async_smem();                // generic-proxy stores of h -> visible to the tensor core
                mbar_arrive(&sh->h_ready[g]);
            }
            if (g == 0 && t == 0) LSTM_TRACE(6, s);
        }
    }
}

template <int KS, int NT, typename TO>
static void lstm_tc_go(dim3 grid, size_t smem, cudaStream_t st, const void* whh, const void* gin, const float* bias_pad, void* hout,
                       const aero_lstm_params& p, const LstmTcShape& sp) {
    const __half* w = static_cast<const __half*>(whh);
    constexpr int kThreads = LstmTcCfg<KS>::kThreads;
    if (p.flags & AERO_TG_A_F16) {          // gate pre-activations stored in FP16
        cudaFuncSetAttribute(lstm_tc_kernel<KS, NT, TO, __half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        lstm_tc_kernel<KS, NT, TO, __half><<<grid, kThreads, smem, st>>>(w, static_cast<const __half*>(gin), bias_pad,
                                                                         static_cast<TO*>(hout), p, sp.S, sp.tps);
    } else {
        cudaFuncSetAttribute(lstm_tc_kernel<KS, NT, TO, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        lstm_tc_kernel<KS, NT, TO, float><<<grid, kThreads, smem, st>>>(w, static_cast<const float*>(gin), bias_pad,
                                                                        static_cast<TO*>(hout), p, sp.S, sp.tps);
    }
}

template <int KS>
static void lstm_tc_dispatch(dim3 grid, cudaStream_t st, const void* whh, const void* gin, const float* bias_pad, void* hout,
                             const aero_lstm_params& p, const LstmTcShape& sp) {
    const size_t smem = 1024 + 2 * (size_t)((KS + 3) / 4) * sp.nt * 128 + 2 * (size_t)sp.nt * LstmTcCfg<KS>::kLdr * 4 + sizeof(LstmTcShared);
    const bool o16 = p.flags & AERO_TG_OUT_F16;
    constexpr int kWide = KS == 6 ? 8 : 16;      // lstm_tc_shape never picks N = 16 at KS = 6
    if (sp.nt == 8) {
        if (o16) lstm_tc_go<KS, 8, __half>(grid, smem, st, whh, gin, bias_pad, hout, p, sp);
        else lstm_tc_go<KS, 8, float>(grid, smem, st, whh, gin, bias_pad, hout, p, sp);
    } else {
        if (o16) lstm_tc_go<KS, kWide, __half>(grid, smem, st, whh, gin, bias_pad, hout, p, sp);
        else lstm_tc_go<KS, kWide, float>(grid, smem, st, whh, gin, bias_pad, hout, p, sp);
    }
}

// Launch shape.  A CTA holds W_hh once (registers of its MMA warpgroups) and two groups of S sequences of one direction, one CTA
// per SM.  A sequence takes tps = ceil((H / 2) / kItems) cell threads, so a group of 128 holds at most 128 / tps sequences
// (8 at H = 96, 16 at H = 48).  S is the smallest width that puts every CTA of both directions on the GPU in one wave,
// ceil(n_seq / (2 floor(sms / 2))), capped there and at 16 (8 for H > 80); beyond the cap the grid takes more than one wave.
// wgmma N = 8 for S <= 8, else 16.
LstmTcShape lstm_tc_shape(int n_seq, int H, int num_sms) {
    LstmTcShape r;
    r.tps = cdiv(H / 2, kItems);
    const int per_dir = std::max(1, num_sms / 2);
    // two MMA warpgroups (H > 80) leave 128 registers per thread: wgmma N = 16 would spill there, so S <= 8
    const int cap = std::min((H + 15) / 16 == 6 ? 8 : 16, kCellThreads / r.tps);
    r.S = std::max(1, std::min(cap, cdiv(n_seq, 2 * per_dir)));
    r.nt = r.S <= 8 ? 8 : 16;
    r.ctas_per_dir = cdiv(n_seq, 2 * r.S);
    return r;
}

int lstm_tc_launch(const void* gin, const float* bias_pad, const void* whh_r, void* hout, const aero_lstm_params& p,
                   cudaStream_t st) {
    const int H = p.H;
    if (H % 4 || H <= 32 || H > 96) {
        set_error("aero_lstm_rec_fwd(wgmma): hidden size %d unsupported (multiple of 4 in (32, 96])", H);
        return AERO_ERR_UNSUPPORTED;
    }
    static int num_sms = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    const int n_seq = p.rows * p.n_win;
    const LstmTcShape sp = lstm_tc_shape(n_seq, H, num_sms);
    const int64_t max_rows = (int64_t)n_seq * p.steps > (int64_t)p.rows * p.T ? (int64_t)n_seq * p.steps : (int64_t)p.rows * p.T;
    if ((max_rows + p.steps) * (8ll * H) >= (1ll << 31)) {
        set_error("aero_lstm_rec_fwd(wgmma): problem too large for 32-bit offsets (%lld rows)", (long long)max_rows);
        return AERO_ERR_UNSUPPORTED;
    }
    const dim3 grid(sp.ctas_per_dir, 2);
    switch ((H + 15) / 16) {
        case 3: lstm_tc_dispatch<3>(grid, st, whh_r, gin, bias_pad, hout, p, sp); break;
        case 4: lstm_tc_dispatch<4>(grid, st, whh_r, gin, bias_pad, hout, p, sp); break;
        case 5: lstm_tc_dispatch<5>(grid, st, whh_r, gin, bias_pad, hout, p, sp); break;
        default: lstm_tc_dispatch<6>(grid, st, whh_r, gin, bias_pad, hout, p, sp); break;
    }
    return check_launch("aero_lstm_rec_fwd(wgmma)");
}

}  // namespace aero

extern "C" int aero_lstm_tc_shape(int32_t n_seq, int32_t H, int32_t num_sms, int32_t* out) {
    if (!out || n_seq < 1 || H % 4 || H <= 32 || H > 96 || num_sms < 1) return AERO_ERR_INVALID;
    const aero::LstmTcShape r = aero::lstm_tc_shape(n_seq, H, num_sms);
    out[0] = r.S;
    out[1] = r.nt;
    out[2] = r.ctas_per_dir;
    out[3] = r.tps;
    return AERO_OK;
}
