// Persistent BiLSTM recurrence on the Hopper tensor cores (wgmma, sm_90a).  See include/aero_b200.h (aero_lstm_rec_fwd,
// precision = 1).
//
// Per step the recurrent term is the small GEMM  D[gate rows x sequences] = W_hh[gate rows x H] * h^T[H x sequences]:
//   A = W_hh, loaded ONCE by TMA into shared memory (K-major, SWIZZLE_128B) and resident for all steps.
//       Gate rows are re-ordered into 128-row M tiles so that a thread finds the gates it needs in its
//       own accumulator row (or one xor-16 shuffle away):
//         GPT = 1 (64 < H <= 128): tile g holds gate g, lane = cell             -> 4 tiles, no exchange
//         GPT = 2 (32 < H <=  64): tile t holds gates (2t, 2t+1); in every warp lanes 0-15 carry gate 2t
//                                  and lanes 16-31 gate 2t+1 of the same 16 cells -> 2 tiles, one shfl.xor 16
//   B = h of the previous step, written by the cell-update threads straight into the swizzled
//       shared-memory operand layout, 16 sequences per CTA;
//   operands are FP16 (K = 16 per wgmma): h is in (-1, 1) and W_hh is O(1), so FP16's 10-bit mantissa gives
//       the same rounding as TF32 at half the shared-memory traffic and half the instruction count; accumulation is fp32;
//   D = (4/GPT) tiles of 128 rows x 16 fp32 columns: the MMA warpgroup holds them in registers (two m64n16 accumulators per
//       tile), writes them to a padded shared-memory tile and the cell-update threads read their row back.
// The input-projection gate pre-activations keep PyTorch's [dir][i,f,g,o][H] column order (a warp reads the contiguous
// cells of one gate per sequence); with one CTA per SM (GPT = 1) they are requested a whole step ahead.
// A CTA owns SEQ = 8 or 16 sequences (the wgmma N stays 16; unused operand rows are zero).  With 8, W_hh for 64 < H <= 96 is
// held in 32-column SWIZZLE_64B chunks (96 KB instead of 128 KB, no zero K padding: 3/4 of the wgmmas per step) and the
// sequences spread over twice as many SMs; for H <= 64 two CTAs share an SM and one CTA's MMA / barrier latency overlaps
// the other's exp-heavy cell update.
// Warps 0..3 are the MMA warpgroup (warp 0 also loads W_hh) and issue the wgmmas from step-invariant descriptors; two mbarriers ping-pong between
// "h ready" and "accumulators ready".  c stays in registers for the whole sequence.  8 (GPT = 2) or 16 (GPT = 1)
// cell-update warps; in the two-gates-per-tile layout a lane finishes only its own half of the warp's sequences.
#include <cuda_fp16.h>
#include <cstdlib>
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

constexpr int kNT = 16;          // wgmma N (operand rows of h); a CTA fills SEQ = 8 or 16 of them
constexpr int kLdAcc = kNT + 4;  // row stride (floats) of the staged accumulators: lane-per-row 16-byte reads hit distinct banks

// tuning knob, read from the environment once: AERO_LSTM_SEQ = 8 / 16 forces the CTA size (0 / unset: chosen per launch)
static int lstm_seq_knob() {
    static const int v = [] { const char* e = getenv("AERO_LSTM_SEQ"); return e ? atoi(e) : 0; }();
    return v;
}

struct LstmTcShared {
    uint64_t w_full;
    uint64_t acc_ready;
    uint64_t h_ready;
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

template <typename T> __device__ __forceinline__ T to_storage(float v);
template <> __device__ __forceinline__ float to_storage<float>(float v) { return v; }
template <> __device__ __forceinline__ __half to_storage<__half>(float v) { return __float2half_rn(v); }

// GPT: gates per 128-row tile.  NEW: cell-update warps (NEW/4 per 32-row quarter of a tile, each owning 4*SEQ/NEW sequences).
// SEQ: sequences per CTA (8 or 16).  ROWB: bytes of K per operand row of a chunk (128 = 64 fp16, SWIZZLE_128B; 64 = 32 fp16,
// SWIZZLE_64B).  MINB: CTAs per SM the register budget is set for.
template <int GPT, int NEW, int SEQ, int ROWB, int MINB, typename TO, typename TG>
__global__ void __launch_bounds__(128 + 32 * NEW, MINB)
lstm_tc_kernel(const __grid_constant__ CUtensorMap mapW, const TG* __restrict__ gin, const float* __restrict__ bias_pad,
               TO* __restrict__ hout, const aero_lstm_params p, const int nK) {
    constexpr int NM = 4 / GPT;                          // M tiles
    constexpr int CPW = 32 / GPT;                        // cells per warp
    constexpr int kNS = 4 * SEQ / NEW;                   // sequences per cell-update warp
    constexpr int kATile = 128 * ROWB, kBTile = kNT * ROWB, kKC = ROWB / 2;   // bytes per A / B chunk tile, fp16 of K per chunk
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sA = smem;                                  // [NM][nK] tiles of 128 rows x ROWB bytes
    uint8_t* sB = smem + NM * nK * kATile;               // [nK] tiles of 16 rows x ROWB bytes
    float* sAcc = reinterpret_cast<float*>(sB + nK * kBTile);   // [NM][128][kLdAcc] staged accumulators
    LstmTcShared* sh = reinterpret_cast<LstmTcShared*>(sAcc + NM * 128 * kLdAcc);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.y;
    const int seq0 = blockIdx.x * SEQ;
    const int n_seq = p.rows * p.n_win;
    const int H = p.H;
    const int ldg = 8 * H;                               // floats per gin row: [dir][i,f,g,o][H], PyTorch's own order

    if (threadIdx.x == 0) {
        mbar_init(&sh->w_full, 1);
        mbar_init(&sh->acc_ready, 128);
        mbar_init(&sh->h_ready, 32 * NEW);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < nK * kBTile / 4; i += blockDim.x) reinterpret_cast<float*>(sB)[i] = 0.f;
    fence_proxy_async_smem();
    __syncthreads();

    if (warp < 4) {
        if (threadIdx.x == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&mapW) : "memory");
            mbar_expect_tx(&sh->w_full, (uint32_t)(NM * nK * kATile));
            for (int m = 0; m < NM; ++m)
                for (int kc = 0; kc < nK; ++kc)
                    tma_load_2d(sA + (m * nK + kc) * kATile, &mapW, &sh->w_full, kc * kKC, (dir * NM + m) * 128);
        }
        // MMA warpgroup.  Every descriptor is step-invariant, so they are built once; only the low bits change along K
        // (+2 per 32 bytes) and with the 64-row half of a tile.
        constexpr int kMaxKC = (ROWB == 128) ? 2 : 4;     // H <= 128
        uint64_t da[NM][kMaxKC], db[kMaxKC];
        const uint32_t a0 = smem_u32(sA), b0 = smem_u32(sB);
#pragma unroll
        for (int kc = 0; kc < kMaxKC; ++kc) {
            db[kc] = make_desc_kmajor<ROWB>(b0 + (uint32_t)(kc * kBTile));
#pragma unroll
            for (int m = 0; m < NM; ++m) da[m][kc] = make_desc_kmajor<ROWB>(a0 + (uint32_t)((m * nK + kc) * kATile));
        }
        float* const arow = sAcc + (warp * 16 + (lane >> 2)) * kLdAcc + 2 * (lane & 3);
        mbar_wait(&sh->w_full, 0);
        for (int s = 1; s < p.steps; ++s) {
            mbar_wait(&sh->h_ready, (uint32_t)((s - 1) & 1));
            LSTM_TRACE(0, s);
            float d[NM][2][8];          // first written by the first wgmma of each chain (scale-d = 0)
            wgmma_fence();
#pragma unroll
            for (int m = 0; m < NM; ++m) {
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
                    for (int kc = 0; kc < kMaxKC; ++kc) {
                        if (kc < nK) {
#pragma unroll
                            for (int k = 0; k < ROWB / 32; ++k)        // K = 16 fp16 = 32 B per wgmma
                                Wgmma<kNT, true, 0>::ss(d[m][hf], da[m][kc] + (uint64_t)(hf * ((64 * ROWB) >> 4) + 2 * k), db[kc] + 2 * k,
                                                        (kc == 0 && k == 0) ? 0u : 1u);
                        }
                    }
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int m = 0; m < NM; ++m)
#pragma unroll
                for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        float* r = arow + (m * 128 + hf * 64) * kLdAcc + 8 * j;
                        *reinterpret_cast<float2*>(r) = make_float2(d[m][hf][4 * j], d[m][hf][4 * j + 1]);
                        *reinterpret_cast<float2*>(r + 8 * kLdAcc) = make_float2(d[m][hf][4 * j + 2], d[m][hf][4 * j + 3]);
                    }
            mbar_arrive(&sh->acc_ready);
            LSTM_TRACE(1, s);
        }
    } else {
        // ===================================================== cell update (warps 4..4+NEW)
        const int ew = warp - 4;
        const int q = warp & 3;                          // 32-row quarter of every tile
        const int wp = ew >> 2;                          // which slice of the 16 sequences
        const int sub = lane / CPW;                      // gate slot inside the tile (0 for GPT=1)
        const int cell = q * CPW + (lane % CPW);
        const bool cell_ok = cell < H;
        const int r = q * 32 + lane;                     // accumulator row == gin column inside a tile
        const int half = p.win_stride / 2;
        const int dpos = dir ? -1 : 1;
        const int pos0 = dir ? p.steps - 1 : 0;

        // Per-sequence state, all loop-invariant work hoisted (32-bit element offsets; the host checks they fit).
        // A step s reads the input projection iff (unsigned)(s - g_lo) < g_len (else the frame is zero padding: bias only)
        // and writes its output iff (unsigned)(s - w_lo) < w_len (window crop of modules.py:53-59 and the T limit).
        // For GPT=2 lane<16 updates even local sequences, lane>=16 odd ones.
        // A lane reads gate pre-activations for all kNS sequences of its warp, but finishes (cell state, h, stores) only
        // kMS = kNS / GPT of them: sequence i = ii*GPT + sub (GPT == 2: the partner lane xor 16 finishes the others).
        // gate pre-activation column of this lane in tile 0 (tile m adds m * GPT * H): gate = m*GPT + sub, this lane's cell
        // (clamped for the padding lanes of the last cells: their values are never used)
        const int gcol = dir * 4 * H + sub * H + min(cell, H - 1);
        const int gtile = GPT * H;
        constexpr int kMS = kNS / GPT;
        int goff[kNS], g_lo[kNS], g_len[kNS];
        int ooff[kMS], w_lo[kMS], w_len[kMS];
        uint32_t baddr[kMS];
        const int jq = (cell & (kKC - 1)) >> 3;                              // 16-byte unit of this cell inside its chunk row
        const uint32_t bbase = smem_u32(sB) + (uint32_t)((cell / kKC) * kBTile + ((cell & 7) << 1));
#pragma unroll
        for (int i = 0; i < kNS; ++i) {
            const int n = wp * kNS + i;
            const int sq = min(seq0 + n, n_seq - 1);
            const int row = sq / p.n_win, k = sq - row * p.n_win;
            const int f0 = k * p.win_stride;                               // first frame of the window
            goff[i] = (p.in_windowed ? (sq * p.steps + pos0) : (row * p.T + f0 + pos0)) * ldg + gcol;
            // valid input positions of this window: frames < T.  position -> step: dir 0: s = pos; dir 1: s = steps-1-pos
            const int in_hi = p.in_windowed ? p.steps : max(0, min(p.steps, p.T - f0));
            g_lo[i] = dir ? p.steps - in_hi : 0;
            g_len[i] = in_hi;
        }
#pragma unroll
        for (int ii = 0; ii < kMS; ++ii) {
            const int n = wp * kNS + ii * GPT + sub;
            const int sq = min(seq0 + n, n_seq - 1);
            const bool exists = seq0 + n < n_seq;
            const int row = sq / p.n_win, k = sq - row * p.n_win;
            const int f0 = k * p.win_stride;
            ooff[ii] = (p.out_windowed ? (sq * p.steps + pos0) : (row * p.T + f0 + pos0)) * 2 * H + dir * H + cell;
            // kept output positions [lo, hi) (window crop of modules.py:53-59) intersected with frames < T
            int lo = 0, hi = p.steps;
            if (!p.out_windowed) {
                lo = (k == 0) ? 0 : half;
                hi = min((k == p.n_win - 1) ? p.steps : p.steps - half, p.T - f0);
            }
            if (!exists || !cell_ok) hi = lo;
            w_lo[ii] = dir ? p.steps - hi : lo;
            w_len[ii] = max(0, hi - lo);
            // swizzled B-operand address of (sequence n, k = cell), fp16: chunk tile cell / kKC, row n (ROWB bytes), 16-byte unit
            // jq XOR-ed with the row (SWIZZLE_128B: n % 8; SWIZZLE_64B: (n / 2) % 4)
            baddr[ii] = bbase + (uint32_t)((n >> 3) * (8 * ROWB) + (n & 7) * ROWB + ((jq ^ (ROWB == 128 ? (n & 7) : ((n >> 1) & 3))) << 4));
        }
        const float* bptr = bias_pad + gcol;
        const int gstep = dpos * ldg, ostep = dpos * 2 * H;

        float c_state[kMS];
#pragma unroll
        for (int i = 0; i < kMS; ++i) c_state[i] = 0.f;

        // The input-projection gate pre-activations stream from HBM (hundreds of MB per layer); their ~1 us load latency must
        // not sit on the per-step dependency chain.  GPT == 1 (one CTA per SM, registers to spare): step s+1's values are
        // requested at the top of step s and consumed a whole step later.  GPT == 2 (two CTAs per SM, register-tight): the
        // loads stay at the top of their own step, but step s+1's lines are pulled into L2 a step ahead.
        constexpr bool kRegPrefetch = (GPT == 1);
        // (kept in the storage type: converting an FP16 value at load time would make the load's result a dependency of the
        // same step and forfeit the step of latency hiding)
        TG gn[kRegPrefetch ? NM : 1][kRegPrefetch ? kNS : 1];
        const TG* const bptr_g = nullptr;
        (void)bptr_g;
        if (kRegPrefetch) {
#pragma unroll
            for (int i = 0; i < kNS; ++i) {
                const bool real = (unsigned)(0 - g_lo[i]) < (unsigned)g_len[i];
#pragma unroll
                for (int m = 0; m < NM; ++m) gn[kRegPrefetch ? m : 0][kRegPrefetch ? i : 0] = real ? gin[goff[i] + m * gtile] : to_storage<TG>(bptr[m * gtile]);
                goff[i] += gstep;
            }
        }
        for (int s = 0; s < p.steps; ++s) {
            float gi[NM][kNS];
            if (kRegPrefetch) {
#pragma unroll
                for (int i = 0; i < kNS; ++i) {
#pragma unroll
                    for (int m = 0; m < NM; ++m) gi[m][i] = ldf(&gn[kRegPrefetch ? m : 0][kRegPrefetch ? i : 0]);
                }
                if (s + 1 < p.steps) {
#pragma unroll
                    for (int i = 0; i < kNS; ++i) {
                        const bool real = (unsigned)(s + 1 - g_lo[i]) < (unsigned)g_len[i];
#pragma unroll
                        for (int m = 0; m < NM; ++m) gn[kRegPrefetch ? m : 0][kRegPrefetch ? i : 0] = real ? gin[goff[i] + m * gtile] : to_storage<TG>(bptr[m * gtile]);
                        goff[i] += gstep;
                    }
                }
            } else {
#pragma unroll
                for (int i = 0; i < kNS; ++i) {
                    const bool real = (unsigned)(s - g_lo[i]) < (unsigned)g_len[i];
#pragma unroll
                    for (int m = 0; m < NM; ++m) gi[m][i] = real ? ldf(gin + goff[i] + m * gtile) : bptr[m * gtile];
                    goff[i] += gstep;
                }
            }
            if (ew == 0 && lane == 0) LSTM_TRACE(2, s);
            if (s > 0) {
                mbar_wait(&sh->acc_ready, (uint32_t)((s - 1) & 1));
            }
            if (ew == 0 && lane == 0) LSTM_TRACE(3, s);
            float a[NM][kNS];
#pragma unroll
            for (int m = 0; m < NM; ++m) {
                uint32_t acc[kNS];
                if (s > 0) {
                    const uint32_t arow = smem_u32(sAcc + (m * 128 + r) * kLdAcc + wp * kNS);
#pragma unroll
                    for (int i = 0; i < kNS; i += 4) {
                        const float4 v = lds128(arow + 4u * i);
                        acc[i] = __float_as_uint(v.x); acc[i + 1] = __float_as_uint(v.y); acc[i + 2] = __float_as_uint(v.z); acc[i + 3] = __float_as_uint(v.w);
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < kNS; ++i) acc[i] = 0u;
                }
                // PyTorch gate order 0 i, 1 f, 2 g, 3 o; gate 2 is tanh = 2*sigmoid(2x) - 1: fold into scale / affine
                const int gate = m * GPT + sub;
                const float k_in = (gate == 2) ? -2.885390081777927f : -1.4426950408889634f;   // -(1|2) * log2(e)
                const float k_mul = (gate == 2) ? 2.0f : 1.0f, k_add = (gate == 2) ? -1.0f : 0.0f;
#pragma unroll
                for (int i = 0; i < kNS; ++i) {
                    const float x = __uint_as_float(acc[i]) + gi[m][i];
                    a[m][i] = fmaf(k_mul, fast_rcp(1.0f + fast_ex2(k_in * x)), k_add);
                }
            }
            if (ew == 0 && lane == 0) LSTM_TRACE(4, s);
#pragma unroll
            for (int ii = 0; ii < kMS; ++ii) {
                float ig, fg, gg, og;
                if (GPT == 1) {
                    ig = a[0][ii]; fg = a[1 % NM][ii]; gg = a[2 % NM][ii]; og = a[3 % NM][ii];
                } else {
                    // this lane finishes sequence 2*ii + sub and hands its two gates of sequence 2*ii + (1 - sub) to the partner
                    const int e = (2 * ii) % kNS, o = (2 * ii + 1) % kNS;
                    const float own0 = sub ? a[0][o] : a[0][e], own1 = sub ? a[1 % NM][o] : a[1 % NM][e];
                    const float snd0 = sub ? a[0][e] : a[0][o], snd1 = sub ? a[1 % NM][e] : a[1 % NM][o];
                    const float p0 = __shfl_xor_sync(0xffffffffu, snd0, 16);
                    const float p1 = __shfl_xor_sync(0xffffffffu, snd1, 16);
                    if (sub == 0) { ig = own0; gg = own1; fg = p0; og = p1; }
                    else          { fg = own0; og = own1; ig = p0; gg = p1; }
                }
                const float c = fmaf(fg, c_state[ii], ig * gg);
                c_state[ii] = c;
                const float th = fmaf(2.0f, fast_rcp(1.0f + fast_ex2(-2.885390081777927f * c)), -1.0f);
                const float h = round_tf32_rna(og * th);
                if (cell_ok) {
                    const unsigned short hh = __half_as_ushort(__float2half_rn(h));
                    asm volatile("st.shared.u16 [%0], %1;" ::"r"(baddr[ii]), "h"(hh) : "memory");
                }
                if ((unsigned)(s - w_lo[ii]) < (unsigned)w_len[ii]) stf(hout + ooff[ii], h);
                ooff[ii] += ostep;
            }
            if (ew == 0 && lane == 0) LSTM_TRACE(5, s);
            if (s + 1 < p.steps) {
                fence_proxy_async_smem();                // generic-proxy stores of h -> visible to the tensor core
                mbar_arrive(&sh->h_ready);
            }
            if (ew == 0 && lane == 0) LSTM_TRACE(6, s);
        }
    }
}

template <int GPT, int NEW, int SEQ, int ROWB, int MINB, typename TO>
static void lstm_tc_go(dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& mW, const void* gin, const float* bias_pad, void* hout,
                       const aero_lstm_params& p, int nK) {
    if (p.flags & AERO_TG_A_F16) {          // gate pre-activations stored in FP16
        cudaFuncSetAttribute(lstm_tc_kernel<GPT, NEW, SEQ, ROWB, MINB, TO, __half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        lstm_tc_kernel<GPT, NEW, SEQ, ROWB, MINB, TO, __half><<<grid, 128 + 32 * NEW, smem, st>>>(mW, static_cast<const __half*>(gin), bias_pad,
                                                                                              static_cast<TO*>(hout), p, nK);
    } else {
        cudaFuncSetAttribute(lstm_tc_kernel<GPT, NEW, SEQ, ROWB, MINB, TO, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        lstm_tc_kernel<GPT, NEW, SEQ, ROWB, MINB, TO, float><<<grid, 128 + 32 * NEW, smem, st>>>(mW, static_cast<const float*>(gin), bias_pad,
                                                                                             static_cast<TO*>(hout), p, nK);
    }
}

int lstm_tc_launch(const void* gin, const float* bias_pad, const void* whh_r, void* hout, const aero_lstm_params& p,
                   cudaStream_t st) {
    const int H = p.H;
    if (H % 4 || H <= 32 || H > 128) {
        set_error("aero_lstm_rec_fwd(wgmma): hidden size %d unsupported (multiple of 4 in (32, 128])", H);
        return AERO_ERR_UNSUPPORTED;
    }
    static int num_sms = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    const int n_seq = p.rows * p.n_win;
    const int gpt = H <= 64 ? 2 : 1;
    const int nM = 4 / gpt;
    const int Kp = ((H + 63) / 64) * 64;                 // the host pads W_hh rows to a multiple of 64 fp16 (128 bytes)
    // Small CTAs (8 sequences) whenever all of them fit on the GPU at once at the co-residency they allow: twice the SMs
    // busy and, where two share an SM (GPT = 2), one CTA's barrier / MMA latency hides behind another's cell update.
    // GPT = 1 keeps W_hh in 32-column SWIZZLE_64B chunks then (no K padding).
    const int knob = lstm_seq_knob();
    const bool small = knob ? knob == 8 : (int64_t)cdiv(n_seq, 8) * 2 <= (int64_t)num_sms * (gpt == 1 ? 1 : 2);
    const int rowb = (gpt == 1 && small) ? 64 : 128;
    const int kc_elems = rowb / 2;
    const int nK = (H + kc_elems - 1) / kc_elems;
    CUtensorMap mW;
    uint64_t dims[2] = {(uint64_t)Kp, (uint64_t)(2 * nM * 128)};
    uint64_t strides[1] = {(uint64_t)Kp * 2};
    uint32_t box[2] = {(uint32_t)kc_elems, 128};
    int rc = encode_map(&mW, whh_r, 2, dims, strides, box, rowb == 64 ? 2 : 0, 2);
    if (rc != AERO_OK) return rc;
    const size_t smem = (size_t)nM * nK * 128 * rowb + (size_t)nK * kNT * rowb + (size_t)nM * 128 * kLdAcc * 4 + sizeof(LstmTcShared) + 1024;
    if (smem > 227 * 1024) {
        set_error("aero_lstm_rec_fwd(wgmma): hidden size %d needs %zu bytes of shared memory", H, smem);
        return AERO_ERR_UNSUPPORTED;
    }
    const int64_t max_rows = (int64_t)n_seq * p.steps > (int64_t)p.rows * p.T ? (int64_t)n_seq * p.steps : (int64_t)p.rows * p.T;
    if ((max_rows + p.steps) * (8ll * H) >= (1ll << 31)) {
        set_error("aero_lstm_rec_fwd(wgmma): problem too large for 32-bit offsets (%lld rows)", (long long)max_rows);
        return AERO_ERR_UNSUPPORTED;
    }
    dim3 grid(cdiv(n_seq, small ? 8 : kNT), 2);
    const bool o16 = p.flags & AERO_TG_OUT_F16;
#define AERO_LSTM_GO(GPT, NEW, SEQ, ROWB, MINB)                                                              \
    do {                                                                                                      \
        if (o16) lstm_tc_go<GPT, NEW, SEQ, ROWB, MINB, __half>(grid, smem, st, mW, gin, bias_pad, hout, p, nK); \
        else lstm_tc_go<GPT, NEW, SEQ, ROWB, MINB, float>(grid, smem, st, mW, gin, bias_pad, hout, p, nK);      \
    } while (0)
    if (gpt == 1) {
        if (small) AERO_LSTM_GO(1, 8, 8, 64, 1);
        else AERO_LSTM_GO(1, 16, 16, 128, 1);
    } else {
        if (small) AERO_LSTM_GO(2, 8, 8, 128, 2);
        else AERO_LSTM_GO(2, 8, 16, 128, 2);
    }
#undef AERO_LSTM_GO
    return check_launch("aero_lstm_rec_fwd(wgmma)");
}

}  // namespace aero
