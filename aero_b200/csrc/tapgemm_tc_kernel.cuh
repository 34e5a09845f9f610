#pragma once
// Kernel of the tap-GEMM on the Hopper tensor cores (sm_90a; host side in tapgemm_tc.cu): TMA -> shared memory -> wgmma (f16 / tf32 operands, fp32 accumulate in
// registers) -> accumulator tile staged in shared memory -> epilogue.  Implicit GEMM, im2col-free: every tap of a convolution
// is a shifted TMA box of the channels-last activation tensor; image borders, channel tails and the K tail are TMA
// out-of-bounds zero fill.
//
//   A tile : 128 pixels (consecutive t of one (b, f) row) x 128 bytes of channels = 128 rows, SWIZZLE_128B
// One translation unit per tile width BN (tapgemm_tc_bn*.cu): the width is a template parameter because the accumulators of
// every width a kernel could run would otherwise be allocated side by side and ptxas would serialise the wgmmas.
//   B tile : BN <= 256 output columns x 128 bytes of channels (weights stored K-major [slab][N][K]) = BN rows
//   D      : two warpgroups x (64 rows x BN fp32 columns) in registers
// Narrow widths (BN <= 128) stage the whole accumulator tile in shared memory at once; the wide ones (192, 256: FP16 operands
// only) stage and finish it kSliceBN columns at a time, so the staging tile stays at 128 x (kSliceBN + 4) floats and three
// 48 KB pipeline stages still fit.
// Persistent CTAs (one per SM) of three warpgroups: warp 0 of the first = TMA producer (runs ahead across tiles); the other
// two each own 64 rows of the tile: they issue the wgmmas of the main loop, write their accumulators to a padded
// shared-memory tile and then run the epilogue on it with two warps per 32-row quarter.  STAGES-deep mbarrier ring between
// the producer and the two consumers; a consumer frees a stage when the wgmmas that read it have retired.
//
// Operand kinds: tf32 (fp32 storage, 32 channels per 128-byte row, K = 8 per wgmma) or f16 (FP16 storage, 64 channels
// per row, K = 16 per wgmma): the shared-memory image is identical in bytes (128 rows x 128 B per k-block, four wgmmas of 32 B along
// K), so one kernel serves both.  FP16 has TF32's 10-bit mantissa at half the HBM bytes and twice the tensor-core rate.
// Outputs are fp32 or FP16 independently of the operand kind.
//
// TF32 operands are read as fp32 bit patterns with the low 13 mantissa bits ignored by the tensor core,
// so producers round activations to TF32 (round-to-nearest) when they store them and the host
// rounds the weights when it packs them: truncation would bias every dot product low.
#include <cuda.h>
#include <type_traits>

#include "tapgemm.cuh"
#include "tc_common.cuh"


namespace aero {

template <bool F16A> struct OperandKind { static constexpr int kBK = F16A ? 64 : 32; };   // elements per 128-byte swizzle row

// number of (tap, source, channel-chunk) iterations and their enumeration, shared by all roles
struct TapIter {
    int fi, dt, slab;
};
__device__ __forceinline__ bool tap_geometry(const aero_tapgemm_params& p, int tap, int fo, TapIter& it) {
    if (p.mode == AERO_TAPS_CONV) {
        const int jf = tap / p.kt, jt = tap - jf * p.kt;
        it.fi = fo * p.stride_f + jf - p.pad_f;
        it.dt = jt * p.dil_t - p.pad_t;
        it.slab = tap;
    } else {
        const int fof = fo + p.f_out_offset;
        it.fi = fof / p.stride_f - tap;
        it.dt = 0;
        it.slab = fof % p.stride_f + tap * p.stride_f;
    }
    return it.fi >= 0 && it.fi < p.F_in;
}

struct TileCoord {
    int b, fo, t0, n0, n_iters;
};
// exact n / d for n < 2^31 (Granlund-Montgomery round-up multiplier, set up by the host): three instructions instead of ~25
__device__ __forceinline__ int fast_div(int n, uint32_t mul, uint32_t shr) {
    return (int)(((uint64_t)(uint32_t)n * mul) >> shr);
}
// number of taps whose input row exists (time-axis borders are TMA zero fill and always count)
__device__ __forceinline__ int valid_taps(const aero_tapgemm_params& p, int fo, int ntaps) {
    if (p.mode == AERO_TAPS_CONV) {
        const int base = fo * p.stride_f - p.pad_f;                    // fi = base + jf
        const int lo = max(0, -base), hi = min(p.kf - 1, p.F_in - 1 - base);
        return max(0, hi - lo + 1) * p.kt;
    }
    const int a = (fo + p.f_out_offset) / p.stride_f;                  // fi = a - tap
    const int lo = max(0, a - p.F_in + 1), hi = min(ntaps - 1, a);
    return max(0, hi - lo + 1);
}
// tile order: the n-tiles of one pixel tile are adjacent, so CTAs working at the same time share the A operand in L2
__device__ __forceinline__ TileCoord tile_coord(const TapGemmArgs& g, int tile, int n_tiles, int BN, int nch1, int nch2) {
    const aero_tapgemm_params& p = g.p;
    TileCoord c;
    if (p.flags & AERO_TG_REVERSE) tile = g.last_tile - tile;       // walk from the end: see AERO_TG_REVERSE
    const int mt = fast_div(tile, g.dv_mul[0], g.dv_shr[0]), nt = tile - mt * n_tiles;
    const int row = fast_div(mt, g.dv_mul[1], g.dv_shr[1]), tt = mt - row * g.tiles_t;
    c.b = fast_div(row, g.dv_mul[2], g.dv_shr[2]);
    c.fo = row - c.b * p.F_out;
    c.t0 = tt * kBM;
    c.n0 = nt * BN;
    c.n_iters = (p.mode == AERO_TAPS_MIX) ? nch1 : valid_taps(p, c.fo, g.ntaps) * (nch1 + nch2);
    return c;
}

// Coalesced epilogue, specialised at compile time (AMODE: 0 none, 1 GELU, 2 ReLU, 3 GLU, 4 LeakyReLU(0.2); RES: residual add; STATS).
// Stage A: this thread's 16 accumulator columns of its row -> bias -> activation / GLU -> row `lane` of the per-warp
// staging tile.  Stage B: the warp walks the tile so that consecutive lanes hold consecutive float4s of one output row
// (residual loads and stores are whole 32-byte sectors of one row), adds the row-wise terms, rounds, accumulates statistics.
template <int AMODE>
__device__ __forceinline__ void epilogue_stage_a(const uint32_t (&r)[16], uint32_t stg_row, uint32_t sbias) {
    // stg_row: shared-space address of this lane's staging row; sbias: shared-space address of this chunk's 16 bias values
    float4 bv[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) bv[j] = lds128(sbias + 16 * j);
#pragma unroll
    for (int j = 0; j < 16; j += 4) {
        float v[4] = {__uint_as_float(r[j]) + bv[j / 4].x, __uint_as_float(r[j + 1]) + bv[j / 4].y,
                      __uint_as_float(r[j + 2]) + bv[j / 4].z, __uint_as_float(r[j + 3]) + bv[j / 4].w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (AMODE == 1) v[u] = gelu_exact(v[u]);
            else if (AMODE == 2) v[u] = fmaxf(v[u], 0.f);
            else if (AMODE == 4) v[u] = leaky_f(v[u]);
        }
        if (AMODE == 3) {
            sts64(stg_row + (j / 2) * 4, v[0] * sigmoid_f(v[1]), v[2] * sigmoid_f(v[3]));
        } else {
            sts128(stg_row + j * 4, make_float4(v[0], v[1], v[2], v[3]));
        }
    }
}

template <int AMODE, bool RES, bool STATS, typename TO>
__device__ __forceinline__ void epilogue_fast_tile(TcShared* sh, const TapGemmArgs& g, const TileCoord& tc, uint32_t tacc, int c_lo, int c_hi,
                                                   int q, int ew, int lane, int Nout, int gw, int c_start, int c_step, uint32_t sbias) {
    const aero_tapgemm_params& p = g.p;
    constexpr int CNT = (AMODE == 3) ? 8 : 16;          // staged output columns per 16 accumulator columns
    constexpr int LPR = CNT / 4;                         // lanes per row (one float4 each)
    constexpr int RPI = 32 / LPR;                        // rows per pass
    const uint32_t stg = smem_u32(&sh->stage[ew][0][0]);       // [32][20] floats, addressed in the shared window
    const bool rnd = (p.flags & 1) && sizeof(TO) == 4;
    float sa = 1.f, sb = 0.f;
    if (g.samp_affine) { sa = g.samp_affine[2 * tc.b]; sb = g.samp_affine[2 * tc.b + 1]; }
    const int cq = lane % LPR, ro = lane / LPR;
    const int row0 = tc.t0 + q * 32;                     // first output row (t) of this warp's lane quarter
    const int rows = min(32, p.T - row0);                // valid rows (<= 0: nothing to store)
    const int g_lo = ((AMODE == 3) ? tc.n0 >> 1 : tc.n0) / gw;
    TO* const obase = static_cast<TO*>(g.out) + (int64_t)tc.b * p.o_sb + (int64_t)tc.fo * p.o_sf + (int64_t)row0 * p.o_st;
    const TO* const rbase = RES ? static_cast<const TO*>(g.residual) + (int64_t)tc.b * p.r_sb + (int64_t)tc.fo * p.r_sf + (int64_t)row0 * p.r_st : nullptr;
    const float* const adp = g.addend_fn ? g.addend_fn + (int64_t)tc.fo * Nout : nullptr;
    for (int c0 = c_lo + c_start; c0 < c_hi; c0 += c_step) {   // split mode: the two warps of a lane quarter alternate 16-column chunks
        const int nb = tc.n0 + c0;
        if (nb >= p.N) break;
        uint32_t r[16];
        if (tc.n_iters > 0) {
            acc_ld16(tacc + 4u * (uint32_t)(c0 - c_lo), r);
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) r[j] = 0u;
        }
        epilogue_stage_a<AMODE>(r, stg + (uint32_t)lane * 80u, sbias + (uint32_t)nb * 4u);
        __syncwarp();
        const int no0 = (AMODE == 3) ? nb >> 1 : nb;
        const int nn = no0 + 4 * cq;
        float ls = 0.f, lq = 0.f;
        if (nn < Nout) {                                 // Nout % 4 == 0 (vec_o)
            float4 ad = make_float4(0.f, 0.f, 0.f, 0.f);
            const bool has_ad = adp != nullptr, affine = g.samp_affine != nullptr;
            if (has_ad) ad = *reinterpret_cast<const float4*>(adp + nn);
            uint32_t sp = stg + (uint32_t)(ro * 80 + cq * 16);
            TO* op = obase + (int64_t)ro * p.o_st + nn;
            const TO* rp = RES ? rbase + (int64_t)ro * p.r_st + nn : nullptr;
            const int64_t ostep = (int64_t)RPI * p.o_st, rstep = (int64_t)RPI * p.r_st;
#pragma unroll 2
            for (int rr = ro; rr < rows; rr += RPI) {
                float4 x = lds128(sp);
                sp += RPI * 80;
                if (has_ad) { x.x += ad.x; x.y += ad.y; x.z += ad.z; x.w += ad.w; }
                if (RES) {
                    const float4 rs = ld4(rp);
                    x.x += rs.x; x.y += rs.y; x.z += rs.z; x.w += rs.w;
                    rp += rstep;
                }
                if (affine) { x.x = fmaf(x.x, sa, sb); x.y = fmaf(x.y, sa, sb); x.z = fmaf(x.z, sa, sb); x.w = fmaf(x.w, sa, sb); }
                if (rnd) { x.x = round_tf32_rna(x.x); x.y = round_tf32_rna(x.y); x.z = round_tf32_rna(x.z); x.w = round_tf32_rna(x.w); }
                if (STATS) {
                    if (sizeof(TO) == 2) {               // statistics describe the values as stored (FP16 pre-normalisation tensors)
                        x.x = stored(x.x, op); x.y = stored(x.y, op); x.z = stored(x.z, op); x.w = stored(x.w, op);
                    }
                    ls += (x.x + x.y) + (x.z + x.w);
                    lq += (x.x * x.x + x.y * x.y) + (x.z * x.z + x.w * x.w);
                }
                st4(op, x);
                op += ostep;
            }
        }
        if (STATS) {
            const int g_first = no0 / gw, g_last = (min(no0 + CNT, Nout) - 1) / gw;
            if (g_first == g_last) {
                // the whole chunk is one group: plain warp reduction (fixed xor order -> deterministic)
                const float a = warp_sum(ls), c = warp_sum(lq);
                if (lane == 0) { sh->stats[ew][g_first - g_lo][0] += a; sh->stats[ew][g_first - g_lo][1] += c; }
            } else {
                // lanes with the same column quad first, then a fixed-order pass over the quads by lane 0
                for (int o = LPR; o < 32; o <<= 1) { ls += __shfl_xor_sync(0xffffffffu, ls, o); lq += __shfl_xor_sync(0xffffffffu, lq, o); }
                if (lane < LPR) { sh->part[ew][lane][0] = ls; sh->part[ew][lane][1] = lq; }
                __syncwarp();
                if (lane == 0) {
                    for (int u = 0; u < LPR; ++u) {
                        const int nq = no0 + 4 * u;
                        if (nq < Nout) {
                            sh->stats[ew][nq / gw - g_lo][0] += sh->part[ew][u][0];
                            sh->stats[ew][nq / gw - g_lo][1] += sh->part[ew][u][1];
                        }
                    }
                }
            }
        }
        __syncwarp();
    }
}

// Direct epilogue: a lane's 16 accumulator columns of its row are 32 (FP16) or 64 (fp32) contiguous bytes -- whole sectors --
// so the row is written straight from registers with 16-byte stores and no shared-memory transpose.  Everything is unrolled
// and independent (bias / residual / addend loads issue together), which is what the HBM-bound layers need: with one or two
// warps per scheduler the epilogue is a latency chain, not a throughput problem.
template <int AMODE, bool RES, bool STATS, typename TO>
__device__ __forceinline__ void epilogue_direct(TcShared* sh, const TapGemmArgs& g, const TileCoord& tc, uint32_t tacc, int c_lo, int c_hi, int q,
                                                int ew, int lane, int Nout, int gw, int c_start, int c_step, uint32_t sbias) {
    const aero_tapgemm_params& p = g.p;
    constexpr int CNT = (AMODE == 3) ? 8 : 16;          // output columns per 16 accumulator columns
    constexpr bool F16 = sizeof(TO) == 2;
    const int t = tc.t0 + q * 32 + lane;
    const bool row_ok = t < p.T;
    TO* const orow = static_cast<TO*>(g.out) + (int64_t)tc.b * p.o_sb + (int64_t)tc.fo * p.o_sf + (int64_t)t * p.o_st;
    const TO* const rrow = RES ? static_cast<const TO*>(g.residual) + (int64_t)tc.b * p.r_sb + (int64_t)tc.fo * p.r_sf + (int64_t)t * p.r_st : nullptr;
    const float* const adp = g.addend_fn ? g.addend_fn + (int64_t)tc.fo * Nout : nullptr;
    float sa = 1.f, sb = 0.f;
    const bool affine = g.samp_affine != nullptr;
    if (affine) { sa = g.samp_affine[2 * tc.b]; sb = g.samp_affine[2 * tc.b + 1]; }
    const bool rnd = (p.flags & 1) && !F16;
    const int g_lo = ((AMODE == 3) ? tc.n0 >> 1 : tc.n0) / gw;
    int cur_g = -1;                                      // statistics: running group (warp-uniform), flushed when it changes
    float ssum = 0.f, ssq = 0.f;
    for (int c0 = c_lo + c_start; c0 < c_hi; c0 += c_step) {
        const int nb = tc.n0 + c0;
        if (nb >= p.N) break;
        uint32_t r[16];
        if (tc.n_iters > 0) {
            acc_ld16(tacc + 4u * (uint32_t)(c0 - c_lo), r);
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) r[j] = 0u;
        }
        float v[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(r[j]);
        {
            float4 bv[4];                                // bias lives in shared memory (zero padded): broadcast reads, no L1 misses
#pragma unroll
            for (int j = 0; j < 4; ++j) bv[j] = lds128(sbias + (uint32_t)nb * 4u + 16u * j);
#pragma unroll
            for (int j = 0; j < 4; ++j) { v[4 * j] += bv[j].x; v[4 * j + 1] += bv[j].y; v[4 * j + 2] += bv[j].z; v[4 * j + 3] += bv[j].w; }
        }
        float o[CNT];
        if (AMODE == 3) {
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = v[2 * j] * sigmoid_f(v[2 * j + 1]);
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j)
                o[j] = (AMODE == 1) ? gelu_exact(v[j]) : (AMODE == 2) ? fmaxf(v[j], 0.f) : (AMODE == 4) ? leaky_f(v[j]) : v[j];
        }
        const int no0 = (AMODE == 3) ? nb >> 1 : nb;
        const int n_ok = min(CNT, Nout - no0);           // valid output columns of this chunk (a multiple of 4; 8 for FP16: host check)
        if (row_ok) {
            if (adp) {
#pragma unroll
                for (int j = 0; j < CNT; j += 4)
                    if (j < n_ok) {
                        const float4 a = __ldg(reinterpret_cast<const float4*>(adp + no0 + j));
                        o[j] += a.x; o[j + 1] += a.y; o[j + 2] += a.z; o[j + 3] += a.w;
                    }
            }
            if (RES) {
#pragma unroll
                for (int j = 0; j < CNT; j += 4)
                    if (j < n_ok) {
                        const float4 a = ld4(rrow + no0 + j);
                        o[j] += a.x; o[j + 1] += a.y; o[j + 2] += a.z; o[j + 3] += a.w;
                    }
            }
            if (affine) {
#pragma unroll
                for (int j = 0; j < CNT; ++j) o[j] = fmaf(o[j], sa, sb);
            }
            if (rnd) {
#pragma unroll
                for (int j = 0; j < CNT; ++j) o[j] = round_tf32_rna(o[j]);
            }
            if (F16 && STATS) {                          // statistics describe the values as stored
#pragma unroll
                for (int j = 0; j < CNT; ++j) o[j] = stored(o[j], orow);
            }
            if (F16) {
#pragma unroll
                for (int j = 0; j < CNT; j += 8)
                    if (j < n_ok) {
                        uint4 u;
                        u.x = pack_half2_sat(o[j], o[j + 1]); u.y = pack_half2_sat(o[j + 2], o[j + 3]);
                        u.z = pack_half2_sat(o[j + 4], o[j + 5]); u.w = pack_half2_sat(o[j + 6], o[j + 7]);
                        *reinterpret_cast<uint4*>(orow + no0 + j) = u;
                    }
            } else {
#pragma unroll
                for (int j = 0; j < CNT; j += 4)
                    if (j < n_ok) *reinterpret_cast<float4*>(orow + no0 + j) = make_float4(o[j], o[j + 1], o[j + 2], o[j + 3]);
            }
        }
        if (STATS) {
            // group width is a multiple of 4 (host check), so every column quad lies in one group
#pragma unroll
            for (int j = 0; j < CNT; j += 4) {
                if (j < n_ok) {
                    const int gi = (no0 + j) / gw;
                    if (gi != cur_g) {
                        if (cur_g >= 0) {
                            const float a = warp_sum(ssum), c = warp_sum(ssq);
                            if (lane == 0) { sh->stats[ew][cur_g - g_lo][0] += a; sh->stats[ew][cur_g - g_lo][1] += c; }
                        }
                        cur_g = gi; ssum = 0.f; ssq = 0.f;
                    }
                    if (row_ok) {
                        ssum += (o[j] + o[j + 1]) + (o[j + 2] + o[j + 3]);
                        ssq += (o[j] * o[j] + o[j + 1] * o[j + 1]) + (o[j + 2] * o[j + 2] + o[j + 3] * o[j + 3]);
                    }
                }
            }
        }
    }
    if (STATS && cur_g >= 0) {
        const float a = warp_sum(ssum), c = warp_sum(ssq);
        if (lane == 0) { sh->stats[ew][cur_g - g_lo][0] += a; sh->stats[ew][cur_g - g_lo][1] += c; }
    }
}

// Main loop of one tile for one consumer warpgroup (rows 64 wg .. 64 wg + 63): n_iters pipeline stages of four wgmmas each into
// the accumulators d.  A stage is handed back to the producer when the wgmmas reading it have retired: one group stays in
// flight, so stage i - 1 is released after the wgmmas of stage i are issued.
template <int BN, bool F16A>
__device__ __forceinline__ void tile_mainloop(TcShared* sh, uint8_t* smem, int& stage, uint32_t& phase, const int kStages, const int stage_bytes,
                                              const int n_iters, const bool mix, const int wg, float (&d)[BN / 2]) {
    const int tid = threadIdx.x & 127, wl = tid >> 5, lane = tid & 31;
    int prev = -1;
    for (int i = 0; i < n_iters; ++i) {
        mbar_wait(&sh->full[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * stage_bytes);
        const uint64_t db = make_desc_sw128(sa + kATileBytes);
        wgmma_fence();
        if (mix && F16A) {
            // MN-major f16 A (transposed-A wgmma), SWIZZLE_128B: atoms of 64 elements along M (128 B) x 8 rows along K = 1024 B.
            // A 64(m) x 64(k) TMA box is 8 K-atoms stacked (SBO = 1024 B) and is this warpgroup's 64 rows; one wgmma
            // (K = 16) consumes two K atoms = 2048 B.
            if constexpr (F16A) {
                const uint32_t sw = sa + (uint32_t)wg * 8192u;
                const uint64_t da = (uint64_t)((sw >> 4) & 0x3FFF) | ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
#pragma unroll
                for (int k = 0; k < 4; ++k) Wgmma<BN, true, 1>::ss(d, da + (uint64_t)(k * (2048 >> 4)), db + 2 * k, (i > 0 || k > 0) ? 1u : 0u);
            }
        } else if (mix) {
            // MN-major tf32 A: wgmma takes tf32 operands from shared memory K-major only, so A goes through registers.  The stage
            // holds four 32(m) x 32(k) TMA boxes (row = k, 128 B of m, SWIZZLE_128B: 16-byte unit ^ (k % 8)); a thread loads
            // its m16n8k8 A fragment (rows g, g + 8; columns c, c + 4) of the warp's 16 rows.
            if constexpr (!F16A) {
                const int m = wg * 64 + wl * 16 + (lane >> 2), c = lane & 3;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    uint32_t a[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int mm = m + (u & 1) * 8, kk = 8 * k + c + (u >> 1) * 4;
                        const uint32_t addr = sa + (uint32_t)((mm >> 5) * 4096 + kk * 128 + ((((mm & 31) >> 2) ^ (kk & 7)) << 4) + ((mm & 3) << 2));
                        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(a[u]) : "r"(addr));
                    }
                    Wgmma<BN, false, 0>::rs(d, a, db + 2 * k, (i > 0 || k > 0) ? 1u : 0u);
                }
            }
        } else {
            const uint64_t da = make_desc_sw128(sa + (uint32_t)wg * (64 * 128));
#pragma unroll
            for (int k = 0; k < 4; ++k)                 // one wgmma = 32 bytes along the swizzled row (K = 8 tf32 / 16 f16)
                Wgmma<BN, F16A, 0>::ss(d, da + 2 * k, db + 2 * k, (i > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && tid == 0) mbar_arrive(&sh->empty[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && tid == 0) mbar_arrive(&sh->empty[prev]);
}

// Accumulator columns [s0, s0 + SW) of this warpgroup -> its 64 rows of the staging tile (row stride SW + 4 floats).  s0 must
// be known at compile time after unrolling: d lives in registers.
template <int BN, int SW>
__device__ __forceinline__ void stage_acc(const float (&d)[BN / 2], const int s0, float* acc, const int wg) {
    constexpr int ldacc = SW + 4;
    const int tid = threadIdx.x & 127, wl = tid >> 5, lane = tid & 31;
    float* row = acc + (wg * 64 + wl * 16 + (lane >> 2)) * ldacc + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < SW / 8; ++j) {
        const int jd = s0 / 8 + j;
        *reinterpret_cast<float2*>(row + 8 * j) = make_float2(d[4 * jd], d[4 * jd + 1]);
        *reinterpret_cast<float2*>(row + 8 * ldacc + 8 * j) = make_float2(d[4 * jd + 2], d[4 * jd + 3]);
    }
}

// Persistent: CTA c processes tiles c, c + gridDim.x, ...  The TMA producer runs ahead across tile boundaries, so the loads of
// tile i+1 are in flight during the epilogue of tile i.
template <int BN, int AMODE, bool RES, bool STATS, bool F16A, bool F16O>
__global__ void __launch_bounds__(kThreads, 1)
tapgemm_tc_kernel(const __grid_constant__ CUtensorMap mapA1, const __grid_constant__ CUtensorMap mapA2,
                  const __grid_constant__ CUtensorMap mapW, const TapGemmArgs g, const int kStages, const int n_tiles,
                  const int tiles_total) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int stage_bytes = kATileBytes + BN * 128;
    TcShared* sh = reinterpret_cast<TcShared*>(smem + kStages * stage_bytes);
    float* const sbias_f = reinterpret_cast<float*>(sh + 1);       // bias (or zeros), padded to whole 16-column chunks of the last tile
    const uint32_t sbias = smem_u32(sbias_f);
    constexpr bool kWide = BN > kMaxBN;
    constexpr int kSW = kWide ? kSliceBN : BN;                     // columns staged at a time
    float* const acc = sbias_f + n_tiles * BN;                     // accumulator staging tile [128][kSW + 4]
    constexpr int ldacc = kSW + 4;                                     // 16-byte rows; lane-per-row 16-byte reads hit distinct banks

    using TO = typename std::conditional<F16O, __half, float>::type;
    constexpr int kBKc = OperandKind<F16A>::kBK;
    const aero_tapgemm_params& p = g.p;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nch1 = (p.C1 + kBKc - 1) / kBKc, nch2 = (p.C2 + kBKc - 1) / kBKc;
    const bool mix = !kWide && p.mode == AERO_TAPS_MIX;         // the host never gives a wide width to the row-mix mode

    for (int i = threadIdx.x; i < n_tiles * BN; i += kThreads) sbias_f[i] = (g.bias && i < g.p.N) ? g.bias[i] : 0.f;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&sh->full[s], 1); mbar_init(&sh->empty[s], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int w = 0; w < kEpiWarps; ++w)
            for (int i = 0; i < 8; ++i) { sh->stats[w][i][0] = 0.f; sh->stats[w][i][1] = 0.f; }
    }
    __syncthreads();

    // wide tiles: the producer warpgroup hands registers to the consumers, whose accumulators take BN / 2 of them
    if (warp < 4) {
        if constexpr (kWide) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
        // ===================================================== TMA producer (warp 0)
        if (warp == 0 && lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA1) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&mapW) : "memory");
            int stage = 0;
            uint32_t phase = 0;
            const uint32_t tx = (uint32_t)stage_bytes;
            int ptl = 0;
            for (int tile = blockIdx.x; tile < tiles_total; tile += gridDim.x, ++ptl) {
                const TileCoord c = tile_coord(g, tile, n_tiles, BN, nch1, nch2);
                if (mix) {
                    // A = activations [K rows][M contiguous].  tf32: four 32(m) x 32(k) boxes, f16: two 64(m) x 64(k) boxes
                    // form one MN-major 128(m) x kBK(k) operand tile of 16 KB
                    for (int kc = 0; kc < nch1; ++kc) {
                        mbar_wait(&sh->empty[stage], phase ^ 1);
                        uint8_t* sa = smem + stage * stage_bytes;
                        mbar_expect_tx(&sh->full[stage], tx);
                        constexpr int kBoxM = F16A ? 64 : 32;
#pragma unroll
                        for (int j = 0; j < 128 / kBoxM; ++j)
                            tma_load_3d(sa + j * (kATileBytes / (128 / kBoxM)), &mapA1, &sh->full[stage], c.t0 + kBoxM * j, kc * kBKc, c.b);
                        tma_load_3d(sa + kATileBytes, &mapW, &sh->full[stage], kc * kBKc, c.n0, 0);
                        if (++stage == kStages) { stage = 0; phase ^= 1; }
                    }
                    continue;
                }
                for (int tap = 0; tap < g.ntaps; ++tap) {
                    TapIter it;
                    if (!tap_geometry(p, tap, c.fo, it)) continue;
                    for (int src = 0; src < 2; ++src) {
                        const int nch = src ? nch2 : nch1;
                        const CUtensorMap* mA = src ? &mapA2 : &mapA1;
                        const int kw0 = src ? p.C1 : 0;
                        for (int kc = 0; kc < nch; ++kc) {
                            mbar_wait(&sh->empty[stage], phase ^ 1);
                            uint8_t* sa = smem + stage * stage_bytes;
                            mbar_expect_tx(&sh->full[stage], tx);
                            tma_load_4d(sa, mA, &sh->full[stage], kc * kBKc, c.t0 + it.dt, it.fi, c.b);
                            tma_load_3d(sa + kATileBytes, &mapW, &sh->full[stage], kw0 + kc * kBKc, c.n0, it.slab);
                            if (++stage == kStages) { stage = 0; phase ^= 1; }
                        }
                    }
                }
            }
        }
    } else {
        if constexpr (kWide) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
        // ===================================================== consumers (warpgroups 1, 2): main loop, then epilogue
        const int wg = (warp >> 2) - 1;                // 64-row half of the tile
        const int ew = warp - 4;                       // epilogue warp index
        const int q = 2 * wg + (warp & 1);             // 32-row quarter of the tile this warp finishes
        const int grp = (warp >> 1) & 1;               // odd / even 16-column chunks
        const int m = q * 32 + lane;
        const int Nout = p.glu ? p.N / 2 : p.N;
        const int gw = (p.stats_mode == 1) ? Nout / p.groups : Nout;
        const bool rnd = (p.flags & 1) && !F16O;
        const int c_start = grp * 16, c_step = 32;
        const bool fast = !mix && g.vec_o && !g.colscale && (p.stats_mode == 0 || gw % 4 == 0);
        int stage = 0, local = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < tiles_total; tile += gridDim.x, ++local) {
            const TileCoord tc = tile_coord(g, tile, n_tiles, BN, nch1, nch2);
            const int b = tc.b, fo = tc.fo, t0 = tc.t0, n0 = tc.n0, n_iters = tc.n_iters;
            const int g_lo = (p.glu ? n0 >> 1 : n0) / gw;
            float d[BN / 2];            // first written by the first wgmma (scale-d = 0); never read when n_iters == 0
            tile_mainloop<BN, F16A>(sh, smem, stage, phase, kStages, stage_bytes, n_iters, mix, wg, d);
            // columns [s0, s0 + kSW) of the tile: staged, then finished by the epilogue (one pass for the narrow widths)
#pragma unroll
            for (int s0 = 0; s0 < BN; s0 += kSW) {
                if (s0 > 0) warpgroup_sync(1 + wg);        // the previous slice is drained
                stage_acc<BN, kSW>(d, s0, acc, wg);
                warpgroup_sync(1 + wg);                    // the staged rows of this half are complete
                const uint32_t tacc = smem_u32(acc + m * ldacc);      // this lane's accumulator row
                const int t = t0 + m;
                const bool row_ok = t < p.T;
                float sa = 1.f, sb = 0.f;
                if (g.samp_affine) { sa = g.samp_affine[2 * b]; sb = g.samp_affine[2 * b + 1]; }
                TO* op = static_cast<TO*>(g.out) + (int64_t)b * p.o_sb + (int64_t)fo * p.o_sf + (int64_t)t * p.o_st;
                const TO* rp = g.residual ? static_cast<const TO*>(g.residual) + (int64_t)b * p.r_sb + (int64_t)fo * p.r_sf + (int64_t)t * p.r_st : nullptr;
                const float* csp = g.colscale ? g.colscale + (int64_t)b * p.cs_sb + (int64_t)t * p.cs_st : nullptr;
                const float* adp = g.addend_fn ? g.addend_fn + (int64_t)fo * Nout : nullptr;
                int cur_g = -1;
                float ssum = 0.f, ssq = 0.f;

                if (mix) {
                    // transposed store: lane = pixel m (contiguous in memory), column = output row n
                    const float gate = (row_ok && g.colscale) ? g.colscale[(int64_t)b * p.cs_sb + t] : 1.f;
                    TO* ob = static_cast<TO*>(g.out) + (int64_t)b * p.o_sb + t;
                    for (int c0 = c_start; c0 < BN; c0 += c_step) {
                        uint32_t r[16];
                        acc_ld16(tacc + 4u * (uint32_t)c0, r);
                        if (row_ok) {
#pragma unroll
                            for (int j = 0; j < 16; ++j) {
                                const int n = n0 + c0 + j;
                                if (n < p.N) {
                                    float x = __uint_as_float(r[j]) * gate;
                                    if (rnd) x = round_tf32_rna(x);
                                    stf(ob + (int64_t)n * p.o_st, x);
                                }
                            }
                        }
                    }
                } else if (fast && (F16O ? (g.vec_o8 && (g.direct_f16 == 1 || (g.direct_f16 == 2 && AMODE == 3))) : g.direct_f32)) {
                    epilogue_direct<AMODE, RES, STATS, TO>(sh, g, tc, tacc, s0, s0 + kSW, q, ew, lane, Nout, gw, c_start, c_step, sbias);
                } else if (fast) {
                    epilogue_fast_tile<AMODE, RES, STATS, TO>(sh, g, tc, tacc, s0, s0 + kSW, q, ew, lane, Nout, gw, c_start, c_step, sbias);
                } else {
                    // generic (unaligned outputs / colscale) epilogue: lane = row, scattered stores; one warp per 32-row quarter
                    for (int c0 = s0; c0 < (grp == 0 ? s0 + kSW : s0); c0 += 16) {
                        uint32_t r[16];
                        if (n_iters > 0) {
                            acc_ld16(tacc + 4u * (uint32_t)(c0 - s0), r);
                        } else {
#pragma unroll
                            for (int j = 0; j < 16; ++j) r[j] = 0u;
                        }
                        const int nb = n0 + c0;
                        if (nb >= p.N) continue;                   // uniform: padded columns of the last tile
                        float v[16];
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int n = nb + j;
                            float x = __uint_as_float(r[j]);
                            if (row_ok && n < p.N) {
                                x += sbias_f[n];
                                if (csp) x *= csp[n];
                                if (p.act == AERO_ACT_GELU) x = gelu_exact(x);
                                else if (p.act == AERO_ACT_RELU) x = fmaxf(x, 0.f);
                                else if (AMODE == 4) x = leaky_f(x);
                            }
                            v[j] = x;
                        }
                        float o[16];
                        int no0, cnt;
                        if (p.glu) {
                            no0 = nb >> 1;
                            cnt = 8;
#pragma unroll
                            for (int j = 0; j < 8; ++j) o[j] = v[2 * j] * sigmoid_f(v[2 * j + 1]);
                        } else {
                            no0 = nb;
                            cnt = 16;
#pragma unroll
                            for (int j = 0; j < 16; ++j) o[j] = v[j];
                        }
                        // statistics bookkeeping is warp-uniform: groups depend on columns only
#pragma unroll
                        for (int sub = 0; sub < 2; ++sub) {
                            if (sub * 8 >= cnt) break;
                            const int ns = no0 + sub * 8;
                            if (p.stats_mode != 0 && ns < Nout) {
                                const int gi = ns / gw;
                                if (gi != cur_g) {
                                    if (cur_g >= 0) {
                                        const float a = warp_sum(ssum), c = warp_sum(ssq);
                                        if (lane == 0) { sh->stats[ew][cur_g - g_lo][0] += a; sh->stats[ew][cur_g - g_lo][1] += c; }
                                    }
                                    cur_g = gi; ssum = 0.f; ssq = 0.f;
                                }
                            }
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                const int jj = sub * 8 + j;
                                const int nn = no0 + jj;
                                if (row_ok && nn < Nout) {
                                    float x = o[jj];
                                    if (adp) x += adp[nn];
                                    if (rp) x += ldf(rp + nn);
                                    x = x * sa + sb;
                                    if (rnd) x = round_tf32_rna(x);
                                    x = stored(x, op);
                                    o[jj] = x;
                                    ssum += x;
                                    ssq += x * x;
                                }
                            }
                        }
                        if (row_ok) {
#pragma unroll
                            for (int j = 0; j < 16; ++j)
                                if (j < cnt && no0 + j < Nout) stf(op + no0 + j, o[j]);
                        }
                    }
                    if (p.stats_mode != 0 && cur_g >= 0) {
                        const float a = warp_sum(ssum), c = warp_sum(ssq);
                        if (lane == 0) { sh->stats[ew][cur_g - g_lo][0] += a; sh->stats[ew][cur_g - g_lo][1] += c; }
                    }
                }
            }
            warpgroup_sync(1 + wg);                    // staging rows drained: the next tile may overwrite them
            if (p.stats_mode != 0) {
                // every warp publishes its own partial sums (fp64 atomics: the order across warps / CTAs only moves the last
                // bits of a double): no CTA-wide barrier on the per-tile path
                __syncwarp();
                if (lane < 8) {
                    const float a = sh->stats[ew][lane][0], c = sh->stats[ew][lane][1];
                    const int gi = g_lo + lane;
                    const int ngroups = (p.stats_mode == 1) ? p.groups : 1;
                    if (gi < ngroups && (a != 0.f || c != 0.f)) {
                        const int64_t slot = (p.stats_mode == 1) ? ((int64_t)b * p.groups + gi) : ((int64_t)b * p.F_out + fo);
                        atomicAdd(&g.stats[2 * slot], (double)a);
                        atomicAdd(&g.stats[2 * slot + 1], (double)c);
                    }
                    sh->stats[ew][lane][0] = 0.f;
                    sh->stats[ew][lane][1] = 0.f;
                }
                __syncwarp();
            }
        }
    }
}



// kernel variants: [operand kind][output type][AMODE][RES][STATS]; only the combinations the host code can produce are
// instantiated for the FP16 kinds (statistics and fp32 outputs go together: GroupNorm inputs stay fp32)
template <int BN, bool F16A, bool F16O>
static KernelFn pick_kernel(int amode, bool res, bool stats) {
#define AERO_TC_K(A, R, S) tapgemm_tc_kernel<BN, A, R, S, F16A, F16O>
    if (amode == 4) return (res || stats) ? nullptr : AERO_TC_K(4, false, false);   // LeakyReLU (SEANet): plain epilogue only
    if constexpr (!F16A && !F16O) {
        static const KernelFn table[4][2][2] = {
            {{AERO_TC_K(0, false, false), AERO_TC_K(0, false, true)}, {AERO_TC_K(0, true, false), AERO_TC_K(0, true, true)}},
            {{AERO_TC_K(1, false, false), AERO_TC_K(1, false, true)}, {AERO_TC_K(1, true, false), AERO_TC_K(1, true, true)}},
            {{AERO_TC_K(2, false, false), AERO_TC_K(2, false, true)}, {AERO_TC_K(2, true, false), AERO_TC_K(2, true, true)}},
            {{AERO_TC_K(3, false, false), AERO_TC_K(3, false, true)}, {AERO_TC_K(3, true, false), AERO_TC_K(3, true, true)}}};
        return table[amode][res][stats];
    } else if constexpr (F16O) {                   // FP16 outputs: statistics / residual only without activation
        if (stats) return (amode == 0 && !res) ? AERO_TC_K(0, false, true) : nullptr;
        if (res) return amode == 0 ? AERO_TC_K(0, true, false) : nullptr;
        switch (amode) {
            case 0: return AERO_TC_K(0, false, false);
            case 1: return AERO_TC_K(1, false, false);
            case 2: return AERO_TC_K(2, false, false);
            default: return AERO_TC_K(3, false, false);
        }
    } else {
        // FP16 operands, fp32 outputs: pre-normalisation outputs (with statistics), LSTM gate inputs, attention q/k/v, FTB gate
        if (res) return nullptr;
        if (stats) return amode == 0 ? AERO_TC_K(0, false, true) : nullptr;
        switch (amode) {
            case 0: return AERO_TC_K(0, false, false);
            case 1: return AERO_TC_K(1, false, false);
            case 2: return AERO_TC_K(2, false, false);
            default: return AERO_TC_K(3, false, false);      // fp32 GLU output: the last decoder layer (feeds the exact-fp32 conv-T)
        }
    }
#undef AERO_TC_K
}

// The kernels of one tile width, chosen by operand kind, output type and epilogue; nullptr when that combination is not built.
// The wide widths are built for FP16 operands only.
template <int BN>
static KernelFn pick_kernel_bn(bool f16a, bool f16o, int amode, bool res, bool stats) {
    if constexpr (BN > kMaxBN)
        return !f16a ? nullptr : f16o ? pick_kernel<BN, true, true>(amode, res, stats) : pick_kernel<BN, true, false>(amode, res, stats);
    else
        return f16a ? (f16o ? pick_kernel<BN, true, true>(amode, res, stats) : pick_kernel<BN, true, false>(amode, res, stats))
                    : (f16o ? pick_kernel<BN, false, true>(amode, res, stats) : pick_kernel<BN, false, false>(amode, res, stats));
}

}  // namespace aero
