// Training-side kernels of the AERO generator (SURVEY.md section 8f rank 1): weight gradients of the tap-GEMM, column
// reductions (bias / BatchNorm statistics / embedding gradients), GroupNorm / BatchNorm + activation forward (training
// form: nothing folded) and backward, fused multi-tensor Adam, operand preparation for the tensor-core modes (weight repack,
// hi / lo TF32 split).  All fp32 storage (the gradient-parity bar is 1e-3 against reference autograd); the tensor-core weight
// gradient lives in wgrad_tc.cu.  Contracts: include/aero_b200.h, "Training".
//
// Data gradients of every convolution are NOT here: the adjoint of a tap-GEMM is a tap-GEMM (flipped taps, transposed
// weights, conv <-> transposed conv), so dgrad runs on aero_tapgemm_fwd itself.
#include <cstdlib>
#include "common.cuh"

namespace aero {

// ------------------------------------------------------------------------------------------------------------ wgrad
// dW[slab][k][n] += sum over output pixels (b, fo, t) of  A(b, fi, t + dt, k) * dY(b, fo, t, n)
// with (fi, dt, slab) the tap geometry of the forward (include/aero_b200.h, aero_tapgemm_fwd).  One CTA: a 128 (k) x 64 (n)
// tile of one slab over a strided subset of 32-pixel chunks (consecutive t of one output row); partial sums are added
// to dW with fp32 atomics (dW is zeroed by the caller).
constexpr int kWgK = 128, kWgP = 32;

struct WgradArgs {
    const float* a1;
    const float* a2;
    const float* dy;
    float* dw;
    aero_tapgemm_params p;
    int64_t dw_sn, dw_sk, dw_ss;      // element strides of dW along n, k, slab
    int tiles_t, k_tiles, n_tiles, vec;
};

// TN = 64: 8 x 4 outputs per thread (narrow layers);  TN = 128: 8 x 8 (the decoder's wide layers: with 8 x 4 the kernel is bound by the
// shared-memory port -- 3 LDS.128 per 32 FMA -- not by the FMA pipe)
template <int TN>
__global__ void __launch_bounds__(256) wgrad_kernel(const WgradArgs g) {
    constexpr int NJ = TN / 16;                        // n outputs per thread
    __shared__ __align__(16) float Xs[kWgP][kWgK];
    __shared__ __align__(16) float Ys[kWgP][TN];
    const aero_tapgemm_params& p = g.p;
    const int K = p.C1 + p.C2;
    const int kt_i = blockIdx.x % g.k_tiles, nt_i = blockIdx.x / g.k_tiles;
    const int k0 = kt_i * kWgK, n0 = nt_i * TN;
    const int slab = blockIdx.y;
    const int tid = threadIdx.x;
    const int ty = tid >> 4, tx = tid & 15;            // micro tile: k = ty*8 .. +7, n = tx*4 .. +3 (and 64 + tx*4 .. for TN = 128)

    // tap geometry of this slab
    int jf = 0, dt = 0, conv_t_r = 0, conv_t_tap = 0;
    if (p.mode == AERO_TAPS_CONV) {
        jf = slab / p.kt;
        dt = (slab - jf * p.kt) * p.dil_t - p.pad_t;
    } else {
        conv_t_r = slab % p.stride_f;
        conv_t_tap = slab / p.stride_f;
    }
    float acc[8][NJ];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;

    const int64_t n_chunks = (int64_t)p.B * p.F_out * g.tiles_t;
    for (int64_t ch = blockIdx.z; ch < n_chunks; ch += gridDim.z) {
        const int tt = (int)(ch % g.tiles_t);
        const int row = (int)(ch / g.tiles_t);
        const int b = row / p.F_out, fo = row - b * p.F_out;
        int fi;
        if (p.mode == AERO_TAPS_CONV) {
            fi = fo * p.stride_f + jf - p.pad_f;
        } else {
            const int fof = fo + p.f_out_offset;
            if (fof % p.stride_f != conv_t_r) continue;
            fi = fof / p.stride_f - conv_t_tap;
        }
        if (fi < 0 || fi >= p.F_in) continue;
        const int t0 = tt * kWgP;
        __syncthreads();
        // ---- load the activation tile [32 pixels][128 channels] and the gradient tile [32][TN]
        for (int i = tid; i < kWgP * (kWgK / 4); i += 256) {
            const int pp = i / (kWgK / 4), c4 = (i - pp * (kWgK / 4)) * 4;
            const int t = t0 + pp, ti = t + dt;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t < p.T && ti >= 0 && ti < p.T_in) {
                const int kk = k0 + c4;
                if (g.vec && kk + 3 < K) {
                    const float* src = (kk < p.C1) ? g.a1 + (int64_t)b * p.a1_sb + (int64_t)fi * p.a1_sf + (int64_t)ti * p.a1_st + kk
                                                   : g.a2 + (int64_t)b * p.a2_sb + (int64_t)fi * p.a2_sf + (int64_t)ti * p.a2_st + (kk - p.C1);
                    v = *reinterpret_cast<const float4*>(src);
                } else {
                    float e[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int kq = kk + u;
                        e[u] = 0.f;
                        if (kq < K)
                            e[u] = (kq < p.C1) ? g.a1[(int64_t)b * p.a1_sb + (int64_t)fi * p.a1_sf + (int64_t)ti * p.a1_st + kq]
                                               : g.a2[(int64_t)b * p.a2_sb + (int64_t)fi * p.a2_sf + (int64_t)ti * p.a2_st + (kq - p.C1)];
                    }
                    v = make_float4(e[0], e[1], e[2], e[3]);
                }
            }
            *reinterpret_cast<float4*>(&Xs[pp][c4]) = v;
        }
        for (int i = tid; i < kWgP * (TN / 4); i += 256) {
            const int pp = i / (TN / 4), c4 = (i - pp * (TN / 4)) * 4;
            const int t = t0 + pp;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t < p.T) {
                const int nn = n0 + c4;
                const float* src = g.dy + (int64_t)b * p.o_sb + (int64_t)fo * p.o_sf + (int64_t)t * p.o_st + nn;
                if (g.vec && nn + 3 < p.N) {
                    v = *reinterpret_cast<const float4*>(src);
                } else {
                    float e[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) e[u] = (nn + u < p.N) ? src[u] : 0.f;
                    v = make_float4(e[0], e[1], e[2], e[3]);
                }
            }
            *reinterpret_cast<float4*>(&Ys[pp][c4]) = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int pp = 0; pp < kWgP; ++pp) {
            const float4 xa = *reinterpret_cast<const float4*>(&Xs[pp][ty * 8]);
            const float4 xb = *reinterpret_cast<const float4*>(&Xs[pp][ty * 8 + 4]);
            const float xs[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
            float ys[NJ];
#pragma unroll
            for (int h = 0; h < NJ / 4; ++h) {
                const float4 yv = *reinterpret_cast<const float4*>(&Ys[pp][h * 64 + tx * 4]);
                ys[4 * h] = yv.x; ys[4 * h + 1] = yv.y; ys[4 * h + 2] = yv.z; ys[4 * h + 3] = yv.w;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < NJ; ++j) acc[i][j] = fmaf(xs[i], ys[j], acc[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int kk = k0 + ty * 8 + i;
        if (kk >= K) continue;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int nn = n0 + (j / 4) * 64 + tx * 4 + (j & 3);
            if (nn < p.N && acc[i][j] != 0.f)
                atomicAdd(g.dw + (int64_t)nn * g.dw_sn + (int64_t)kk * g.dw_sk + (int64_t)slab * g.dw_ss, acc[i][j]);
        }
    }
}

// Thin problems -- a handful of weights against up to a million pixels (the discriminator's 1 -> 16 first layer, the 96 -> 2 last
// transposed convolution, the 2 -> 48 first one, FTB's C -> 5): the 128 x 64 tile above would be almost empty.  Here one thread owns up
// to kWsPer weights (slab, k, n), a CTA owns a run of frames of one output row; validity of the tap's input row is decided once per
// (weight, row), the inner loop over frames is two loads and one FMA.  Partial sums go to dW with fp32 atomics.
constexpr int kWsPer = 8, kWsThreads = 256;

__global__ void __launch_bounds__(kWsThreads) wgrad_small_kernel(const WgradArgs g, int n_out, int n_seg, int seg_len) {
    const aero_tapgemm_params& p = g.p;
    const int K = p.C1 + p.C2, KN = K * p.N;
    int o_n[kWsPer], o_k[kWsPer], o_dt[kWsPer], o_fa[kWsPer];
    float acc[kWsPer];
#pragma unroll
    for (int i = 0; i < kWsPer; ++i) {
        const int o = threadIdx.x + i * kWsThreads;
        acc[i] = 0.f;
        o_n[i] = -1; o_k[i] = 0; o_dt[i] = 0; o_fa[i] = 0;
        if (o < n_out) {
            const int slab = o / KN, rem = o - slab * KN;
            o_k[i] = rem / p.N;
            o_n[i] = rem - o_k[i] * p.N;
            if (p.mode == AERO_TAPS_CONV) {
                const int jf = slab / p.kt;
                o_fa[i] = jf;
                o_dt[i] = (slab - jf * p.kt) * p.dil_t - p.pad_t;
            } else {
                o_fa[i] = slab;                         // residue = slab % stride_f, tap = slab / stride_f
            }
        }
    }
    const int row = blockIdx.x / n_seg, seg = blockIdx.x - row * n_seg;
    const int b = row / p.F_out, fo = row - b * p.F_out;
    const int t_lo = seg * seg_len, t_hi = min(p.T, t_lo + seg_len);
    const float* dyr = g.dy + (int64_t)b * p.o_sb + (int64_t)fo * p.o_sf;
#pragma unroll
    for (int i = 0; i < kWsPer; ++i) {
        if (o_n[i] < 0) continue;
        int fi;
        if (p.mode == AERO_TAPS_CONV) {
            fi = fo * p.stride_f + o_fa[i] - p.pad_f;
        } else {
            const int fof = fo + p.f_out_offset;
            if (fof % p.stride_f != o_fa[i] % p.stride_f) continue;
            fi = fof / p.stride_f - o_fa[i] / p.stride_f;
        }
        if (fi < 0 || fi >= p.F_in) continue;
        const int k = o_k[i], dt = o_dt[i];
        const float* xr;
        int64_t xs;
        if (k < p.C1) { xr = g.a1 + (int64_t)b * p.a1_sb + (int64_t)fi * p.a1_sf + k; xs = p.a1_st; }
        else { xr = g.a2 + (int64_t)b * p.a2_sb + (int64_t)fi * p.a2_sf + (k - p.C1); xs = p.a2_st; }
        const int lo = max(t_lo, -dt), hi = min(t_hi, p.T_in - dt);          // frames whose input frame t + dt exists
        const float* yp = dyr + o_n[i];
        // eight independent load pairs in flight per thread: the loop is bound by L2 latency, not by arithmetic
        float a[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) a[u] = 0.f;
        int t = lo;
        for (; t + 7 < hi; t += 8) {
            float xv[8], yv[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                xv[u] = __ldg(xr + (int64_t)(t + u + dt) * xs);
                yv[u] = __ldg(yp + (int64_t)(t + u) * p.o_st);
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) a[u] = fmaf(xv[u], yv[u], a[u]);
        }
        for (; t < hi; ++t) a[0] = fmaf(__ldg(xr + (int64_t)(t + dt) * xs), __ldg(yp + (int64_t)t * p.o_st), a[0]);
        const float a0 = (a[0] + a[1]) + (a[2] + a[3]), a1 = (a[4] + a[5]) + (a[6] + a[7]);
        acc[i] = a0 + a1;
    }
#pragma unroll
    for (int i = 0; i < kWsPer; ++i) {
        if (o_n[i] < 0 || acc[i] == 0.f) continue;
        const int o = threadIdx.x + i * kWsThreads;
        const int slab = o / KN;
        atomicAdd(g.dw + (int64_t)o_n[i] * g.dw_sn + (int64_t)o_k[i] * g.dw_sk + (int64_t)slab * g.dw_ss, acc[i]);
    }
}

// The same for layers with at most 8 output channels (96 -> 2 transposed convolution, FTB's C -> 5): a thread owns up to four (slab, k)
// pairs and ALL n of them, so that consecutive lanes read consecutive input channels (one 128-byte line per warp and frame) and the few
// gradient values of a frame are one broadcast load for the whole warp.
constexpr int kWtnItems = 4, kWtnN = 8;
__global__ void __launch_bounds__(kWsThreads) wgrad_thin_n_kernel(const WgradArgs g, int n_items, int n_seg, int seg_len) {
    const aero_tapgemm_params& p = g.p;
    const int K = p.C1 + p.C2;
    const int row = blockIdx.x / n_seg, seg = blockIdx.x - row * n_seg;
    const int b = row / p.F_out, fo = row - b * p.F_out;
    const int t_lo = seg * seg_len, t_hi = min(p.T, t_lo + seg_len);
    const float* dyr = g.dy + (int64_t)b * p.o_sb + (int64_t)fo * p.o_sf;
#pragma unroll 1
    for (int i = 0; i < kWtnItems; ++i) {
        const int it = threadIdx.x + i * kWsThreads;
        if (it >= n_items) break;
        const int slab = it / K, k = it - slab * K;
        int fi, dt = 0;
        if (p.mode == AERO_TAPS_CONV) {
            const int jf = slab / p.kt;
            fi = fo * p.stride_f + jf - p.pad_f;
            dt = (slab - jf * p.kt) * p.dil_t - p.pad_t;
        } else {
            const int fof = fo + p.f_out_offset;
            if (fof % p.stride_f != slab % p.stride_f) continue;
            fi = fof / p.stride_f - slab / p.stride_f;
        }
        if (fi < 0 || fi >= p.F_in) continue;
        const float* xr;
        int64_t xs;
        if (k < p.C1) { xr = g.a1 + (int64_t)b * p.a1_sb + (int64_t)fi * p.a1_sf + k; xs = p.a1_st; }
        else { xr = g.a2 + (int64_t)b * p.a2_sb + (int64_t)fi * p.a2_sf + (k - p.C1); xs = p.a2_st; }
        const int lo = max(t_lo, -dt), hi = min(t_hi, p.T_in - dt);
        float acc[kWtnN];
#pragma unroll
        for (int n = 0; n < kWtnN; ++n) acc[n] = 0.f;
        int t = lo;
        for (; t + 3 < hi; t += 4) {                                     // four frames in flight
            float xv[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) xv[u] = __ldg(xr + (int64_t)(t + u + dt) * xs);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float* yp = dyr + (int64_t)(t + u) * p.o_st;
#pragma unroll
                for (int n = 0; n < kWtnN; ++n)
                    if (n < p.N) acc[n] = fmaf(xv[u], __ldg(yp + n), acc[n]);
            }
        }
        for (; t < hi; ++t) {
            const float xv = __ldg(xr + (int64_t)(t + dt) * xs);
            const float* yp = dyr + (int64_t)t * p.o_st;
#pragma unroll
            for (int n = 0; n < kWtnN; ++n)
                if (n < p.N) acc[n] = fmaf(xv, __ldg(yp + n), acc[n]);
        }
        float* out = g.dw + (int64_t)k * g.dw_sk + (int64_t)slab * g.dw_ss;
#pragma unroll
        for (int n = 0; n < kWtnN; ++n)
            if (n < p.N && acc[n] != 0.f) atomicAdd(out + (int64_t)n * g.dw_sn, acc[n]);
    }
}

// ------------------------------------------------------------------------------------------------------------ weight repack
// [taps][K][ldn] (N contiguous: the SIMT tap-GEMM layout) -> [taps][ldn][K] (K contiguous: the wgmma layout), rounded to TF32
// (round-to-nearest, ties away: cvt.rna) -- the training step repacks every weight it uses, every step, so this is one launch instead
// of a transpose, an add and a mask.
__global__ void __launch_bounds__(256) pack_kmajor_tf32_kernel(const float* __restrict__ w, float* __restrict__ out, float* __restrict__ out_lo,
                                                               int K, int ldn) {
    __shared__ float tile[32][33];
    const int tap = blockIdx.z, k0 = blockIdx.x * 32, n0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const float* src = w + (int64_t)tap * K * ldn;
    for (int r = ty; r < 32; r += 8)
        tile[r][tx] = (k0 + r < K && n0 + tx < ldn) ? src[(int64_t)(k0 + r) * ldn + n0 + tx] : 0.f;
    __syncthreads();
    for (int r = ty; r < 32; r += 8)
        if (n0 + r < ldn && k0 + tx < K) {
            const float v = tile[tx][r], hi = round_tf32_rna(v);
            const int64_t o = (int64_t)tap * K * ldn + (int64_t)(n0 + r) * K + k0 + tx;
            out[o] = hi;
            if (out_lo) out_lo[o] = round_tf32_rna(v - hi);          // v - hi is exact in fp32; its TF32 rounding leaves 2^-22 |v|
        }
}

// x = hi + lo with hi = TF32(x) (round to nearest) and lo = TF32(x - hi): the operand split of the 3xTF32 GEMM (three tensor-core products
// hi*hi + hi*lo + lo*hi reproduce the fp32 product to ~2^-22)
__global__ void __launch_bounds__(256) split_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, int64_t n) {
    const int64_t n4 = n >> 2;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (int64_t)gridDim.x * 256) {
        const float4 v = reinterpret_cast<const float4*>(x)[i];
        float4 h, l;
        h.x = round_tf32_rna(v.x); h.y = round_tf32_rna(v.y); h.z = round_tf32_rna(v.z); h.w = round_tf32_rna(v.w);
        l.x = round_tf32_rna(v.x - h.x); l.y = round_tf32_rna(v.y - h.y); l.z = round_tf32_rna(v.z - h.z); l.w = round_tf32_rna(v.w - h.w);
        reinterpret_cast<float4*>(hi)[i] = h;
        reinterpret_cast<float4*>(lo)[i] = l;
    }
    if (blockIdx.x == 0)
        for (int64_t i = (n4 << 2) + threadIdx.x; i < n; i += 256) {
            const float h = round_tf32_rna(x[i]);
            hi[i] = h;
            lo[i] = round_tf32_rna(x[i] - h);
        }
}

// ------------------------------------------------------------------------------------------------------------ gram
// out[i][j] += sum_{b, m} P[b][i][m] * gate[b][m] * Q[b][j][m]   (i, j < F rows; m < M contiguous positions): the weight
// gradient of FTB's frequency mix `freq_fc` (modules.py:296,317-320), whose contraction runs over the CONTIGUOUS axis of two
// channels-last tensors.  64 x 64 output tile per CTA, 32 positions per step, split over (b, m chunks), fp32 atomics.
__global__ void __launch_bounds__(256) gram_kernel(const float* __restrict__ P, const float* __restrict__ Q, const float* __restrict__ gate,
                                                   float* __restrict__ out, int F, int64_t M, int64_t sb_p, int64_t sb_q, int64_t sb_g,
                                                   int chunks_per_b) {
    __shared__ float Ps[32][65], Qs[32][65];
    const int i0 = blockIdx.x * 64, j0 = blockIdx.y * 64;
    const int b = blockIdx.z / chunks_per_b, ck = blockIdx.z % chunks_per_b;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    float acc[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = 0.f;
    const float* Pb = P + (int64_t)b * sb_p;
    const float* Qb = Q + (int64_t)b * sb_q;
    const float* Gb = gate ? gate + (int64_t)b * sb_g : nullptr;
    for (int64_t m0 = (int64_t)ck * 32; m0 < M; m0 += (int64_t)chunks_per_b * 32) {
        __syncthreads();
        for (int e = tid; e < 64 * 32; e += 256) {
            const int r = e >> 5, mm = e & 31;
            const int64_t m = m0 + mm;
            float pv = 0.f, qv = 0.f;
            if (m < M) {
                const float gv = Gb ? Gb[m] : 1.f;
                if (i0 + r < F) pv = Pb[(int64_t)(i0 + r) * M + m] * gv;
                if (j0 + r < F) qv = Qb[(int64_t)(j0 + r) * M + m];
            }
            Ps[mm][r] = pv;
            Qs[mm][r] = qv;
        }
        __syncthreads();
#pragma unroll 8
        for (int mm = 0; mm < 32; ++mm) {
            float pa[4], qa[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) { pa[u] = Ps[mm][ty * 4 + u]; qa[u] = Qs[mm][tx * 4 + u]; }
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int v = 0; v < 4; ++v) acc[u][v] = fmaf(pa[u], qa[v], acc[u][v]);
        }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int i = i0 + ty * 4 + u, j = j0 + tx * 4 + v;
            if (i < F && j < F && acc[u][v] != 0.f) atomicAdd(out + (int64_t)i * F + j, acc[u][v]);
        }
}

// x[b][f][t][c] += addend[f][c]   (frequency embedding, aero.py:475-480, un-fused for training)
__global__ void __launch_bounds__(256) bcast_add_kernel(float* __restrict__ x, const float* __restrict__ addend, int64_t total4, int F, int T,
                                                        int C) {
    const int c4n = C >> 2;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total4; i += (int64_t)gridDim.x * 256) {
        const int c4 = (int)(i % c4n);
        const int f = (int)((i / c4n / T) % F);
        float4 v = reinterpret_cast<float4*>(x)[i];
        const float4 a = reinterpret_cast<const float4*>(addend + (int64_t)f * C)[c4];
        v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
        reinterpret_cast<float4*>(x)[i] = v;
    }
}

// y[b][i] = x[b][i] * s[b * s_stride]   (de-normalisation backward: per-sample scale)
__global__ void __launch_bounds__(256) scale_rows_kernel(const float* __restrict__ x, float* __restrict__ y, const float* __restrict__ s,
                                                         int64_t per_sample, int s_stride) {
    const float k = s[(int64_t)blockIdx.y * s_stride];
    const float* xb = x + (int64_t)blockIdx.y * per_sample;
    float* yb = y + (int64_t)blockIdx.y * per_sample;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < per_sample; i += (int64_t)gridDim.x * 256) yb[i] = xb[i] * k;
}

// ------------------------------------------------------------------------------------------------------------ colsum
// out1[seg][n] += sum_{o < n_outer, i < n_inner} x[seg*seg_sx + o*outer_s + i*inner_s + n]
// out2[seg][n] += the same sum of x * z (z addressed like x); either output may be null.  OUT = float or double.
template <typename OUT>
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, const float* __restrict__ z, OUT* out1, OUT* out2,
                                                     int N, int64_t n_inner, int64_t inner_s, int64_t n_outer, int64_t outer_s,
                                                     int64_t seg_sx, int64_t seg_so) {
    __shared__ float s1[8][32], s2[8][32];
    const int col = blockIdx.x * 32 + threadIdx.x;
    const int seg = blockIdx.z;
    const int64_t rows = n_inner * n_outer;
    float a1 = 0.f, a2 = 0.f;
    if (col < N) {
        const float* xb = x + (int64_t)seg * seg_sx + col;
        const float* zb = z ? z + (int64_t)seg * seg_sx + col : nullptr;
        for (int64_t r = (int64_t)blockIdx.y * 8 + threadIdx.y; r < rows; r += (int64_t)gridDim.y * 8) {
            const int64_t o = r / n_inner, i = r - o * n_inner;
            const int64_t off = o * outer_s + i * inner_s;
            const float v = xb[off];
            a1 += v;
            if (zb) a2 = fmaf(v, zb[off], a2);
        }
    }
    s1[threadIdx.y][threadIdx.x] = a1;
    s2[threadIdx.y][threadIdx.x] = a2;
    __syncthreads();
    if (threadIdx.y == 0 && col < N) {
        float t1 = 0.f, t2 = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) { t1 += s1[k][threadIdx.x]; t2 += s2[k][threadIdx.x]; }
        if (out1) atomicAdd(out1 + (int64_t)seg * seg_so + col, (OUT)t1);
        if (out2) atomicAdd(out2 + (int64_t)seg * seg_so + col, (OUT)t2);
    }
}

// The same reduction for 16-byte-aligned rows (N % 4 == 0): a thread owns 4 columns (one float4 per row), four rows in flight per thread,
// row -> (outer, inner) by carries instead of a 64-bit division per element.  This is the form every bias / statistics gradient of the
// training step takes; it runs at HBM speed where the scalar kernel above reaches a fifth of it.
template <typename OUT>
__global__ void __launch_bounds__(256) colsum4_kernel(const float* __restrict__ x, const float* __restrict__ z, OUT* out1, OUT* out2,
                                                      int N, int64_t n_inner, int64_t inner_s, int64_t n_outer, int64_t outer_s,
                                                      int64_t seg_sx, int64_t seg_so) {
    __shared__ float4 s1[8][32], s2[8][32];
    const int col = (blockIdx.x * 32 + threadIdx.x) * 4;
    const int seg = blockIdx.z;
    const int64_t rows = n_inner * n_outer;
    float4 a1 = make_float4(0.f, 0.f, 0.f, 0.f), a2 = a1;
    if (col < N) {
        const float* xb = x + (int64_t)seg * seg_sx + col;
        const float* zb = z ? z + (int64_t)seg * seg_sx + col : nullptr;
        const int64_t step = (int64_t)gridDim.y * 8;
        int64_t r = (int64_t)blockIdx.y * 8 + threadIdx.y;
        int64_t o = r / n_inner, i = r - o * n_inner;
        const int64_t d_o = step / n_inner, d_i = step - d_o * n_inner;
        auto advance = [&]() {
            r += step; i += d_i; o += d_o;
            if (i >= n_inner) { i -= n_inner; ++o; }
        };
        while (r + 3 * step < rows) {
            float4 v[4], w[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int64_t off = o * outer_s + i * inner_s;
                v[u] = *reinterpret_cast<const float4*>(xb + off);
                if (zb) w[u] = *reinterpret_cast<const float4*>(zb + off);
                advance();
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                a1.x += v[u].x; a1.y += v[u].y; a1.z += v[u].z; a1.w += v[u].w;
                if (zb) { a2.x = fmaf(v[u].x, w[u].x, a2.x); a2.y = fmaf(v[u].y, w[u].y, a2.y); a2.z = fmaf(v[u].z, w[u].z, a2.z); a2.w = fmaf(v[u].w, w[u].w, a2.w); }
            }
        }
        for (; r < rows; advance()) {
            const int64_t off = o * outer_s + i * inner_s;
            const float4 v = *reinterpret_cast<const float4*>(xb + off);
            a1.x += v.x; a1.y += v.y; a1.z += v.z; a1.w += v.w;
            if (zb) {
                const float4 w = *reinterpret_cast<const float4*>(zb + off);
                a2.x = fmaf(v.x, w.x, a2.x); a2.y = fmaf(v.y, w.y, a2.y); a2.z = fmaf(v.z, w.z, a2.z); a2.w = fmaf(v.w, w.w, a2.w);
            }
        }
    }
    s1[threadIdx.y][threadIdx.x] = a1;
    s2[threadIdx.y][threadIdx.x] = a2;
    __syncthreads();
    if (threadIdx.y == 0 && col < N) {
        float4 t1 = make_float4(0.f, 0.f, 0.f, 0.f), t2 = t1;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float4 p1 = s1[k][threadIdx.x], p2 = s2[k][threadIdx.x];
            t1.x += p1.x; t1.y += p1.y; t1.z += p1.z; t1.w += p1.w;
            t2.x += p2.x; t2.y += p2.y; t2.z += p2.z; t2.w += p2.w;
        }
        const float e1[4] = {t1.x, t1.y, t1.z, t1.w}, e2[4] = {t2.x, t2.y, t2.z, t2.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (out1) atomicAdd(out1 + (int64_t)seg * seg_so + col + u, (OUT)e1[u]);
            if (out2) atomicAdd(out2 + (int64_t)seg * seg_so + col + u, (OUT)e2[u]);
        }
    }
}

// ------------------------------------------------------------------------------------------------------------ add
__global__ void __launch_bounds__(256) add_kernel(float* __restrict__ dst, const float* __restrict__ src, int64_t n, float alpha) {
    const int64_t n4 = n >> 2;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (int64_t)gridDim.x * 256) {
        float4 d = reinterpret_cast<float4*>(dst)[i];
        const float4 s = reinterpret_cast<const float4*>(src)[i];
        d.x = fmaf(alpha, s.x, d.x); d.y = fmaf(alpha, s.y, d.y); d.z = fmaf(alpha, s.z, d.z); d.w = fmaf(alpha, s.w, d.w);
        reinterpret_cast<float4*>(dst)[i] = d;
    }
    if (blockIdx.x == 0)
        for (int64_t i = (n4 << 2) + threadIdx.x; i < n; i += 256) dst[i] = fmaf(alpha, src[i], dst[i]);
}

// dst (fp32) += src (fp64): the last step of every bias / affine / statistics gradient (fp64 column sums into the fp32 parameter gradient)
__global__ void __launch_bounds__(256) add_f64_kernel(float* __restrict__ dst, const double* __restrict__ src, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) dst[i] += (float)src[i];
}

// ------------------------------------------------------------------------------------------------------------ norm + act (training)
// y = act(norm(x)):  norm = GroupNorm (scope 1: per sample and channel group over all rows; scope 2: per (b, f) row, one
// group), BatchNorm with batch statistics (scope 3: per channel over every pixel of the batch) or none (AERO_NA_NO_NORM).
// act: AERO_NA_* of the inference kernel plus AERO_NA_RELU.  Thread mapping as in norm_act_kernel: a thread owns one quad
// of OUTPUT channels and walks pixels.
constexpr int kNaMaxGroups = 8;
constexpr int kNaMaxC = 1536;

struct NaConst {        // per-thread constants of its channel quad(s)
    float m[4], r[4], ga[4], be[4];
};

__device__ __forceinline__ void na_load_const(NaConst& k, const aero_norm_act_params& p, const double* stats, const float* gamma,
                                              const float* beta, int seg, int c) {
    const bool nonorm = p.flags & AERO_NA_NO_NORM;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        k.m[u] = 0.f; k.r[u] = 1.f; k.ga[u] = 1.f; k.be[u] = 0.f;
    }
    if (nonorm) return;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        k.ga[u] = gamma[c + u];
        k.be[u] = beta[c + u];
        double n;
        int64_t slot;
        if (p.scope == 1) { n = (double)p.F_in * p.T * (p.C / p.groups); slot = (int64_t)seg * p.groups + (c + u) / (p.C / p.groups); }
        else if (p.scope == 2) { n = (double)p.T * p.C; slot = seg; }
        else { n = (double)p.B * p.F_in * p.T; slot = c + u; }
        const double mean = stats[2 * slot] / n;
        double var = stats[2 * slot + 1] / n - mean * mean;
        if (var < 0) var = 0;
        k.m[u] = (float)mean;
        k.r[u] = (float)(1.0 / sqrt(var + (double)p.eps));
    }
}

// activation value and derivative pieces for one element.  For GLU the caller handles the pair.
__device__ __forceinline__ float na_act(int op, float g, float al) {
    if (op == AERO_NA_GELU) return gelu_exact(g);
    if (op == AERO_NA_RELU) return fmaxf(g, 0.f);
    if (op == AERO_NA_LEAKY) return g > 0.f ? g : 0.2f * g;
    if (op == AERO_NA_TANH) return tanhf(g);
    if (op == AERO_NA_SNAKE) { const float sn = sinf(g * al); return g + sn * sn / al; }
    return g;
}
__device__ __forceinline__ float na_dact(int op, float g, float al) {
    if (op == AERO_NA_GELU) {
        // d/dg [0.5 g (1 + erf(g/sqrt2))] = 0.5 (1 + erf(g/sqrt2)) + g * exp(-g^2/2) / sqrt(2 pi)
        return 0.5f * (1.0f + erff(g * 0.70710678118654752440f)) + g * 0.3989422804014327f * expf(-0.5f * g * g);
    }
    if (op == AERO_NA_RELU) return g > 0.f ? 1.f : 0.f;
    if (op == AERO_NA_LEAKY) return g > 0.f ? 1.f : 0.2f;
    if (op == AERO_NA_TANH) { const float t = tanhf(g); return 1.f - t * t; }
    if (op == AERO_NA_SNAKE) { return 1.0f + sinf(2.0f * g * al); }          // 1 + 2 sin(ag) cos(ag)
    return 1.f;
}

template <int OP>
__global__ void __launch_bounds__(256) na_train_fwd_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           const float* __restrict__ snake_a, const float* __restrict__ scale,
                                                           const float* __restrict__ residual, float* __restrict__ y,
                                                           const aero_norm_act_params p) {
    constexpr bool GLU = (OP == AERO_NA_GLU || OP == AERO_NA_GLU_SCALE_RES);
    const int seg = blockIdx.y;
    const int Cout = GLU ? p.C / 2 : p.C;
    const int c4n = Cout >> 2;
    const int ppp = 256 / c4n;
    const int cq = threadIdx.x % c4n, dp = threadIdx.x / c4n;
    if (dp >= ppp) return;
    const int c = cq * 4;
    int b, f_lo, f_hi;
    if (p.scope == 2) { b = seg / p.F_in; f_lo = seg % p.F_in; f_hi = f_lo + 1; } else { b = seg; f_lo = 0; f_hi = p.F_out; }
    NaConst k0, k1;
    na_load_const(k0, p, stats, gamma, beta, seg, c);
    if (GLU) na_load_const(k1, p, stats, gamma, beta, seg, c + Cout);
    float sc[4] = {1.f, 1.f, 1.f, 1.f};
    if (OP == AERO_NA_GLU_SCALE_RES) {
#pragma unroll
        for (int u = 0; u < 4; ++u) sc[u] = scale[c + u];
    }
    const int64_t npix = (int64_t)(f_hi - f_lo) * p.T;
    for (int64_t pix = (int64_t)blockIdx.x * ppp + dp; pix < npix; pix += (int64_t)gridDim.x * ppp) {
        const int fl = f_lo + (int)(pix / p.T), t = (int)(pix % p.T);
        const float* xp = x + (((int64_t)b * p.F_in + fl + p.f_off) * p.T + t) * p.C + c;
        const int64_t oi = (((int64_t)b * p.F_out + fl) * p.T + t) * Cout + c;
        const float4 v = *reinterpret_cast<const float4*>(xp);
        const float xv[4] = {v.x, v.y, v.z, v.w};
        float o[4];
        if (GLU) {
            const float4 v2 = *reinterpret_cast<const float4*>(xp + Cout);
            const float xw[4] = {v2.x, v2.y, v2.z, v2.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float ga = fmaf((xv[u] - k0.m[u]) * k0.r[u], k0.ga[u], k0.be[u]);
                const float gb = fmaf((xw[u] - k1.m[u]) * k1.r[u], k1.ga[u], k1.be[u]);
                o[u] = ga * sigmoid_f(gb);
            }
            if (OP == AERO_NA_GLU_SCALE_RES) {
                const float4 rs = *reinterpret_cast<const float4*>(residual + oi);
                o[0] = fmaf(sc[0], o[0], rs.x); o[1] = fmaf(sc[1], o[1], rs.y); o[2] = fmaf(sc[2], o[2], rs.z); o[3] = fmaf(sc[3], o[3], rs.w);
            }
        } else {
            const float al = (OP == AERO_NA_SNAKE) ? snake_a[fl + p.f_off] : 1.f;
#pragma unroll
            for (int u = 0; u < 4; ++u) o[u] = na_act(OP, fmaf((xv[u] - k0.m[u]) * k0.r[u], k0.ga[u], k0.be[u]), al);
        }
        *reinterpret_cast<float4*>(y + oi) = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// Backward, pass 1 (APPLY = false): accumulates  dgamma[c] += sum dg * xh,  dbeta[c] += sum dg,  dscale[c] += sum dy * glu,
// dsnake[f] += sum dy * d act / d a,  and the per-(segment, group) sums  ws[slot] += {sum dxh, sum dxh * xh}  (dxh = dg * gamma)
// that the GroupNorm backward needs (scope 1 / 2; BatchNorm derives them from dgamma / dbeta).
// Pass 2 (APPLY = true):  dx = rstd * (dxh - S1/n - xh * S2/n)   (no norm: dx = dg) for every input row (rows outside the
// crop [f_off, f_off + F_out) have dy = 0 but still receive the mean terms).
template <int OP, bool APPLY>
__global__ void __launch_bounds__(256) na_train_bwd_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           const float* __restrict__ snake_a, const float* __restrict__ scale,
                                                           const float* __restrict__ dy, float* __restrict__ dx,
                                                           double* dgamma, double* dbeta, double* dscale, double* dsnake, double* ws,
                                                           const aero_norm_act_params p) {
    constexpr bool GLU = (OP == AERO_NA_GLU || OP == AERO_NA_GLU_SCALE_RES);
    __shared__ float s_dg[APPLY ? 1 : kNaMaxC], s_db[APPLY ? 1 : kNaMaxC], s_ds[APPLY ? 1 : kNaMaxC / 2];
    __shared__ double s_grp[kNaMaxGroups][2];
    __shared__ float s_da;
    const bool nonorm = p.flags & AERO_NA_NO_NORM;
    const int seg = blockIdx.y;
    const int Cout = GLU ? p.C / 2 : p.C;
    const int c4n = Cout >> 2;
    const int ppp = 256 / c4n;
    const int cq = threadIdx.x % c4n, dp = threadIdx.x / c4n;
    if (!APPLY) {
        for (int i = threadIdx.x; i < p.C; i += 256) { s_dg[i] = 0.f; s_db[i] = 0.f; }
        for (int i = threadIdx.x; i < Cout; i += 256) s_ds[i] = 0.f;
        if (threadIdx.x < kNaMaxGroups) { s_grp[threadIdx.x][0] = 0.0; s_grp[threadIdx.x][1] = 0.0; }
        if (threadIdx.x == 0) s_da = 0.f;
        __syncthreads();
    }
    const bool active = dp < ppp;
    const int c = cq * 4;
    int b, f_lo, f_hi;                  // INPUT rows covered by this segment
    if (p.scope == 2) { b = seg / p.F_in; f_lo = seg % p.F_in; f_hi = f_lo + 1; } else { b = seg; f_lo = 0; f_hi = p.F_in; }
    NaConst k0, k1;
    float sc[4] = {1.f, 1.f, 1.f, 1.f};
    float m1a[4] = {0.f, 0.f, 0.f, 0.f}, m2a[4] = {0.f, 0.f, 0.f, 0.f}, m1b[4] = {0.f, 0.f, 0.f, 0.f}, m2b[4] = {0.f, 0.f, 0.f, 0.f};
    if (active) {
        na_load_const(k0, p, stats, gamma, beta, seg, c);
        if (GLU) na_load_const(k1, p, stats, gamma, beta, seg, c + Cout);
        if (OP == AERO_NA_GLU_SCALE_RES) {
#pragma unroll
            for (int u = 0; u < 4; ++u) sc[u] = scale[c + u];
        }
        if (APPLY && !nonorm) {
            // means of dxh and dxh * xh over the normalisation set of each channel
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (p.scope == 3) {
                    const double n = (double)p.B * p.F_in * p.T;
                    m1a[u] = (float)((double)k0.ga[u] * dbeta[c + u] / n);
                    m2a[u] = (float)((double)k0.ga[u] * dgamma[c + u] / n);
                    if (GLU) {
                        m1b[u] = (float)((double)k1.ga[u] * dbeta[c + Cout + u] / n);
                        m2b[u] = (float)((double)k1.ga[u] * dgamma[c + Cout + u] / n);
                    }   // (dgamma / dbeta are the fp64 accumulators of pass 1)
                } else {
                    const int gw = p.C / p.groups;
                    const double n = (p.scope == 1) ? (double)p.F_in * p.T * gw : (double)p.T * p.C;
                    const int64_t sa = (p.scope == 1) ? (int64_t)seg * p.groups + (c + u) / gw : seg;
                    m1a[u] = (float)(ws[2 * sa] / n);
                    m2a[u] = (float)(ws[2 * sa + 1] / n);
                    if (GLU) {
                        const int64_t sb = (p.scope == 1) ? (int64_t)seg * p.groups + (c + Cout + u) / gw : seg;
                        m1b[u] = (float)(ws[2 * sb] / n);
                        m2b[u] = (float)(ws[2 * sb + 1] / n);
                    }
                }
            }
        }
    }
    float adg[4] = {0.f, 0.f, 0.f, 0.f}, adb[4] = {0.f, 0.f, 0.f, 0.f}, bdg[4] = {0.f, 0.f, 0.f, 0.f}, bdb[4] = {0.f, 0.f, 0.f, 0.f};
    float ads[4] = {0.f, 0.f, 0.f, 0.f};
    double g1a = 0.0, g2a = 0.0, g1b = 0.0, g2b = 0.0;
    float da_acc = 0.f;
    const int64_t npix = (int64_t)(f_hi - f_lo) * p.T;
    if (active)
    for (int64_t pix = (int64_t)blockIdx.x * ppp + dp; pix < npix; pix += (int64_t)gridDim.x * ppp) {
        const int fin = f_lo + (int)(pix / p.T), t = (int)(pix % p.T);
        const int fout = fin - p.f_off;
        const bool has_dy = fout >= 0 && fout < p.F_out;
        if (!APPLY && !has_dy) continue;
        const int64_t xi = (((int64_t)b * p.F_in + fin) * p.T + t) * p.C + c;
        const float4 v = *reinterpret_cast<const float4*>(x + xi);
        const float xv[4] = {v.x, v.y, v.z, v.w};
        float dyv[4] = {0.f, 0.f, 0.f, 0.f};
        if (has_dy) {
            const float4 d = *reinterpret_cast<const float4*>(dy + (((int64_t)b * p.F_out + fout) * p.T + t) * Cout + c);
            dyv[0] = d.x; dyv[1] = d.y; dyv[2] = d.z; dyv[3] = d.w;
        }
        float xha[4], dga[4], xhb[4], dgb[4];
        if (GLU) {
            const float4 v2 = *reinterpret_cast<const float4*>(x + xi + Cout);
            const float xw[4] = {v2.x, v2.y, v2.z, v2.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                xha[u] = (xv[u] - k0.m[u]) * k0.r[u];
                xhb[u] = (xw[u] - k1.m[u]) * k1.r[u];
                const float ga = fmaf(xha[u], k0.ga[u], k0.be[u]), gb = fmaf(xhb[u], k1.ga[u], k1.be[u]);
                const float sg = sigmoid_f(gb);
                const float de = dyv[u] * sc[u];
                dga[u] = de * sg;
                dgb[u] = de * ga * sg * (1.0f - sg);
                if (!APPLY && OP == AERO_NA_GLU_SCALE_RES) ads[u] = fmaf(dyv[u], ga * sg, ads[u]);
            }
        } else {
            const float al = (OP == AERO_NA_SNAKE) ? snake_a[fin] : 1.f;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                xha[u] = (xv[u] - k0.m[u]) * k0.r[u];
                const float ga = fmaf(xha[u], k0.ga[u], k0.be[u]);
                dga[u] = dyv[u] * na_dact(OP, ga, al);
                if (!APPLY && OP == AERO_NA_SNAKE) {
                    // d/da [g + sin^2(a g) / a] = g sin(2 a g) / a - sin^2(a g) / a^2
                    const float sn = sinf(al * ga);
                    da_acc = fmaf(dyv[u], ga * sinf(2.0f * al * ga) / al - sn * sn / (al * al), da_acc);
                }
            }
        }
        if (!APPLY) {
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                adb[u] += dga[u];
                adg[u] = fmaf(dga[u], xha[u], adg[u]);
                const float dxh = dga[u] * k0.ga[u];
                g1a += dxh;
                g2a += dxh * xha[u];
                if (GLU) {
                    bdb[u] += dgb[u];
                    bdg[u] = fmaf(dgb[u], xhb[u], bdg[u]);
                    const float dxb = dgb[u] * k1.ga[u];
                    g1b += dxb;
                    g2b += dxb * xhb[u];
                }
            }
        } else {
            float o[4], o2[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (nonorm) {
                    o[u] = dga[u];
                    if (GLU) o2[u] = dgb[u];
                } else {
                    o[u] = k0.r[u] * (dga[u] * k0.ga[u] - m1a[u] - xha[u] * m2a[u]);
                    if (GLU) o2[u] = k1.r[u] * (dgb[u] * k1.ga[u] - m1b[u] - xhb[u] * m2b[u]);
                }
            }
            *reinterpret_cast<float4*>(dx + xi) = make_float4(o[0], o[1], o[2], o[3]);
            if (GLU) *reinterpret_cast<float4*>(dx + xi + Cout) = make_float4(o2[0], o2[1], o2[2], o2[3]);
        }
    }
    if (APPLY) return;
    if (active) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            atomicAdd(&s_dg[c + u], adg[u]);
            atomicAdd(&s_db[c + u], adb[u]);
            if (GLU) { atomicAdd(&s_dg[c + Cout + u], bdg[u]); atomicAdd(&s_db[c + Cout + u], bdb[u]); }
            if (OP == AERO_NA_GLU_SCALE_RES) atomicAdd(&s_ds[c + u], ads[u]);
        }
        if (!nonorm && p.scope != 3) {
            const int gw = p.C / p.groups;
            const int ga_i = (p.scope == 1) ? c / gw : 0;
            atomicAdd(&s_grp[ga_i][0], g1a);
            atomicAdd(&s_grp[ga_i][1], g2a);
            if (GLU) {
                const int gb_i = (p.scope == 1) ? (c + Cout) / gw : 0;
                atomicAdd(&s_grp[gb_i][0], g1b);
                atomicAdd(&s_grp[gb_i][1], g2b);
            }
        }
        if (OP == AERO_NA_SNAKE) atomicAdd(&s_da, da_acc);
    }
    __syncthreads();
    if (!nonorm) {
        for (int i = threadIdx.x; i < p.C; i += 256) {
            if (s_dg[i] != 0.f) atomicAdd(dgamma + i, (double)s_dg[i]);
            if (s_db[i] != 0.f) atomicAdd(dbeta + i, (double)s_db[i]);
        }
        if (p.scope != 3 && threadIdx.x < p.groups) {
            const int64_t slot = (p.scope == 1) ? (int64_t)seg * p.groups + threadIdx.x : seg;
            atomicAdd(ws + 2 * slot, s_grp[threadIdx.x][0]);
            atomicAdd(ws + 2 * slot + 1, s_grp[threadIdx.x][1]);
        }
    }
    if (OP == AERO_NA_GLU_SCALE_RES)
        for (int i = threadIdx.x; i < Cout; i += 256)
            if (s_ds[i] != 0.f) atomicAdd(dscale + i, (double)s_ds[i]);
    if (OP == AERO_NA_SNAKE && threadIdx.x == 0 && s_da != 0.f) atomicAdd(dsnake + f_lo, (double)s_da);
}

// ------------------------------------------------------------------------------------------------------------ Adam
// One launch for every parameter tensor: chunk table [n_chunks] of {param, grad, exp_avg, exp_avg_sq, count}.
// torch.optim.Adam semantics (no amsgrad, no weight decay): m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
// p -= lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps).
struct AdamChunk {
    float* p;
    const float* g;
    float* m;
    float* v;
    int64_t n;
};

__global__ void __launch_bounds__(256) adam_kernel(const AdamChunk* __restrict__ chunks, float lr, float b1, float b2, float eps,
                                                   float bc1, float bc2_sqrt, float grad_scale) {
    const AdamChunk ch = chunks[blockIdx.x];
    const float step = lr / bc1;
    for (int64_t i = threadIdx.x; i < ch.n; i += 256) {
        const float g = ch.g[i] * grad_scale;
        const float m = fmaf(b1, ch.m[i], (1.0f - b1) * g);
        const float v = fmaf(b2, ch.v[i], (1.0f - b2) * g * g);
        ch.m[i] = m;
        ch.v[i] = v;
        ch.p[i] -= step * m / (sqrtf(v) / bc2_sqrt + eps);
    }
}

bool wgrad_tc_eligible(const aero_tapgemm_params& p, const void* a1, const void* a2, const void* dy);
int wgrad_tc_launch(const float* a1, const float* a2, const float* dy, float* dw, const aero_tapgemm_params& p, int64_t dw_sn, int64_t dw_sk,
                    int64_t dw_ss, cudaStream_t st);
}  // namespace aero

// ================================================================================================================ C ABI
extern "C" int aero_tapgemm_wgrad(const float* a1, const float* a2, const float* dy, float* dw, const aero_tapgemm_params* p,
                                  int64_t dw_sn, int64_t dw_sk, int64_t dw_ss, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(dy && dw && p && (a1 || a2), "aero_tapgemm_wgrad: null argument");
    AERO_REQUIRE(p->mode == AERO_TAPS_CONV || p->mode == AERO_TAPS_CONVT, "aero_tapgemm_wgrad: mode %d", p->mode);
    AERO_REQUIRE((p->C1 == 0 || a1) && (p->C2 == 0 || a2) && p->C1 + p->C2 >= 1 && p->N >= 1, "aero_tapgemm_wgrad: channels");
    AERO_REQUIRE(p->mode != AERO_TAPS_CONVT || (p->kt == 1 && p->kf % p->stride_f == 0), "aero_tapgemm_wgrad: transposed-conv geometry");
    if (p->precision == 1 && wgrad_tc_eligible(*p, a1, a2, dy))        // TF32 tensor-core training mode (csrc/wgrad_tc.cu)
        return wgrad_tc_launch(a1, a2, dy, dw, *p, dw_sn, dw_sk, dw_ss, (cudaStream_t)stream);
    WgradArgs g;
    g.a1 = a1; g.a2 = a2; g.dy = dy; g.dw = dw; g.p = *p;
    g.dw_sn = dw_sn; g.dw_sk = dw_sk; g.dw_ss = dw_ss;
    const int K = p->C1 + p->C2;
    g.tiles_t = cdiv(p->T, kWgP);
    // (the 8 x 8 variant, TN = 128, is kept for experiments; it has not been compared on H100, so the narrow one serves all;
    //  AERO_WGRAD_WIDE=1 selects it for experiments)
    static const bool wide = getenv("AERO_WGRAD_WIDE") != nullptr;
    const int TN = (wide && p->N >= 128) ? 128 : 64;
    g.k_tiles = cdiv(K, kWgK);
    g.n_tiles = cdiv(p->N, TN);
    auto al4 = [](int64_t v) { return (v & 3) == 0; };
    g.vec = (p->C1 % 4 == 0) && (p->C2 % 4 == 0) && (p->N % 4 == 0) && al4(p->a1_sb) && al4(p->a1_sf) && al4(p->a1_st) && al4(p->a2_sb) &&
            al4(p->a2_sf) && al4(p->a2_st) && al4(p->o_sb) && al4(p->o_sf) && al4(p->o_st) &&
            ((((uintptr_t)a1 | (uintptr_t)a2 | (uintptr_t)dy) & 15) == 0);
    const int nslab = (p->mode == AERO_TAPS_CONVT) ? p->kf : p->kf * p->kt;
    const int64_t n_chunks = (int64_t)p->B * p->F_out * g.tiles_t;
    if ((int64_t)nslab * K * p->N <= kWsPer * kWsThreads && (int64_t)p->B * p->F_out * p->T >= 4096) {
        // few weights, many pixels: one thread per weight
        const int64_t n_rows = (int64_t)p->B * p->F_out;
        int n_seg = (int)cdiv((int64_t)132 * 8, n_rows);
        if (n_seg > cdiv(p->T, 32)) n_seg = cdiv(p->T, 32);
        if (n_seg < 1) n_seg = 1;
        const int seg_len = cdiv(p->T, n_seg);
        n_seg = cdiv(p->T, seg_len);
        AERO_REQUIRE(n_rows * n_seg <= 2147483647LL, "aero_tapgemm_wgrad: grid too large");
        if (p->N <= kWtnN && K >= 16 && nslab * K <= kWtnItems * kWsThreads) {
            wgrad_thin_n_kernel<<<(unsigned)(n_rows * n_seg), kWsThreads, 0, (cudaStream_t)stream>>>(g, nslab * K, n_seg, seg_len);
            return check_launch("aero_tapgemm_wgrad(thin n)");
        }
        wgrad_small_kernel<<<(unsigned)(n_rows * n_seg), kWsThreads, 0, (cudaStream_t)stream>>>(g, nslab * K * p->N, n_seg, seg_len);
        return check_launch("aero_tapgemm_wgrad(small)");
    }
    // enough CTAs to fill the GPU a few times over, never more than chunks
    int64_t tiles = (int64_t)g.k_tiles * g.n_tiles * nslab;
    int64_t splits = (132 * 6 + tiles - 1) / tiles;
    if (splits > n_chunks) splits = n_chunks;
    if (splits > 65535) splits = 65535;
    if (splits < 1) splits = 1;
    AERO_REQUIRE(nslab <= 65535, "aero_tapgemm_wgrad: too many taps");
    dim3 grid((unsigned)(g.k_tiles * g.n_tiles), (unsigned)nslab, (unsigned)splits);
    if (TN == 128) wgrad_kernel<128><<<grid, 256, 0, (cudaStream_t)stream>>>(g);
    else wgrad_kernel<64><<<grid, 256, 0, (cudaStream_t)stream>>>(g);
    return check_launch("aero_tapgemm_wgrad");
}

extern "C" int aero_pack_kmajor_tf32(const float* w, float* out, float* out_lo, int32_t taps, int32_t K, int32_t ldn, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(w && out && taps >= 1 && taps <= 65535 && K >= 1 && ldn >= 1, "aero_pack_kmajor_tf32: bad argument");
    dim3 grid((unsigned)cdiv(K, 32), (unsigned)cdiv(ldn, 32), (unsigned)taps);
    pack_kmajor_tf32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, out, out_lo, K, ldn);
    return check_launch("aero_pack_kmajor_tf32");
}

extern "C" int aero_split_tf32(const float* x, float* hi, float* lo, int64_t n, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && hi && lo && n >= 1, "aero_split_tf32: bad argument");
    AERO_REQUIRE((((uintptr_t)x | (uintptr_t)hi | (uintptr_t)lo) & 15) == 0, "aero_split_tf32: 16-byte aligned buffers");
    int64_t blocks = (n / 4 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks < 1) blocks = 1;
    split_tf32_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, hi, lo, n);
    return check_launch("aero_split_tf32");
}

extern "C" int aero_tapgemm_wgrad_tc_eligible(const aero_tapgemm_params* p, const float* a1, const float* a2, const float* dy) {
    return p && aero::wgrad_tc_eligible(*p, a1, a2, dy) ? 1 : 0;
}

extern "C" int aero_colsum(const float* x, const float* z, void* out1, void* out2, int32_t out_double, int32_t N, int64_t n_inner,
                           int64_t inner_stride, int64_t n_outer, int64_t outer_stride, int32_t n_seg, int64_t seg_stride_x,
                           int64_t seg_stride_out, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && (out1 || out2) && N >= 1 && n_inner >= 1 && n_outer >= 1 && n_seg >= 1 && n_seg <= 65535, "aero_colsum: bad argument");
    const int64_t rows = n_inner * n_outer;
    if (N % 4 == 0 && inner_stride % 4 == 0 && outer_stride % 4 == 0 && seg_stride_x % 4 == 0 &&
        ((((uintptr_t)x) | ((uintptr_t)z)) & 15) == 0) {
        const int xt = cdiv(N, 128);
        int64_t ys = (rows + 8 * 16 - 1) / (8 * 16);                   // at least 16 rows per thread
        const int64_t cap4 = (int64_t)132 * 8 / ((int64_t)xt * n_seg) + 1;
        if (ys > cap4) ys = cap4;
        if (ys < 1) ys = 1;
        if (ys > 65535) ys = 65535;
        dim3 grid4((unsigned)xt, (unsigned)ys, (unsigned)n_seg), block4(32, 8);
        if (out_double)
            colsum4_kernel<double><<<grid4, block4, 0, (cudaStream_t)stream>>>(x, z, (double*)out1, (double*)out2, N, n_inner, inner_stride,
                                                                              n_outer, outer_stride, seg_stride_x, seg_stride_out);
        else
            colsum4_kernel<float><<<grid4, block4, 0, (cudaStream_t)stream>>>(x, z, (float*)out1, (float*)out2, N, n_inner, inner_stride,
                                                                             n_outer, outer_stride, seg_stride_x, seg_stride_out);
        return check_launch("aero_colsum");
    }
    int64_t ysplit = (rows + 8 * 64 - 1) / (8 * 64);
    const int64_t cap = (int64_t)132 * 16 / (cdiv(N, 32) * (int64_t)n_seg) + 1;
    if (ysplit > cap) ysplit = cap;
    if (ysplit < 1) ysplit = 1;
    if (ysplit > 65535) ysplit = 65535;
    dim3 grid((unsigned)cdiv(N, 32), (unsigned)ysplit, (unsigned)n_seg), block(32, 8);
    if (out_double)
        colsum_kernel<double><<<grid, block, 0, (cudaStream_t)stream>>>(x, z, (double*)out1, (double*)out2, N, n_inner, inner_stride, n_outer,
                                                                       outer_stride, seg_stride_x, seg_stride_out);
    else
        colsum_kernel<float><<<grid, block, 0, (cudaStream_t)stream>>>(x, z, (float*)out1, (float*)out2, N, n_inner, inner_stride, n_outer,
                                                                      outer_stride, seg_stride_x, seg_stride_out);
    return check_launch("aero_colsum");
}

extern "C" int aero_gram(const float* P, const float* Q, const float* gate, float* out, int32_t B, int32_t F, int64_t M, int64_t sb_p,
                         int64_t sb_q, int64_t sb_g, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(P && Q && out && B >= 1 && F >= 1 && M >= 1, "aero_gram: bad argument");
    const int tiles = cdiv(F, 64);
    int chunks = (132 * 4) / (tiles * tiles * B) + 1;
    const int64_t max_chunks = (M + 31) / 32;
    if (chunks > max_chunks) chunks = (int)max_chunks;
    AERO_REQUIRE((int64_t)B * chunks <= 65535, "aero_gram: too many z blocks");
    dim3 grid((unsigned)tiles, (unsigned)tiles, (unsigned)(B * chunks));
    gram_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(P, Q, gate, out, F, M, sb_p, sb_q, sb_g, chunks);
    return check_launch("aero_gram");
}

extern "C" int aero_bcast_add(float* x, const float* addend, int32_t B, int32_t F, int32_t T, int32_t C, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && addend && B >= 1 && F >= 1 && T >= 1 && C >= 4 && C % 4 == 0, "aero_bcast_add: bad argument");
    const int64_t total4 = (int64_t)B * F * T * (C / 4);
    int64_t blocks = (total4 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    bcast_add_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, addend, total4, F, T, C);
    return check_launch("aero_bcast_add");
}

extern "C" int aero_scale_rows(const float* x, float* y, const float* s, int32_t B, int64_t per_sample, int32_t s_stride, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && y && s && B >= 1 && B <= 65535 && per_sample >= 1, "aero_scale_rows: bad argument");
    int64_t blocks = (per_sample + 256 * 8 - 1) / (256 * 8);
    if (blocks > 4096) blocks = 4096;
    dim3 grid((unsigned)blocks, (unsigned)B);
    scale_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, s, per_sample, s_stride);
    return check_launch("aero_scale_rows");
}

extern "C" int aero_add(float* dst, const float* src, int64_t n, float alpha, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(dst && src && n >= 0 && ((((uintptr_t)dst | (uintptr_t)src) & 15) == 0), "aero_add: bad argument");
    if (n == 0) return AERO_OK;
    int64_t blocks = (n / 4 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks < 1) blocks = 1;
    add_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(dst, src, n, alpha);
    return check_launch("aero_add");
}

extern "C" int aero_add_f64(float* dst, const double* src, int64_t n, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(dst && src && n >= 0, "aero_add_f64: bad argument");
    if (n == 0) return AERO_OK;
    int64_t blocks = (n + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    add_f64_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(dst, src, n);
    return check_launch("aero_add_f64");
}

static int na_train_check(const aero_norm_act_params* p) {
    using namespace aero;
    AERO_REQUIRE(p->scope >= 1 && p->scope <= 3, "aero_norm_act_train: scope=%d", p->scope);
    const bool glu = (p->op == AERO_NA_GLU || p->op == AERO_NA_GLU_SCALE_RES);
    const int Cout = glu ? p->C / 2 : p->C;
    AERO_REQUIRE(p->C % 4 == 0 && Cout % 4 == 0 && Cout / 4 <= 256 && p->C <= kNaMaxC, "aero_norm_act_train: C=%d", p->C);
    const bool nonorm = p->flags & AERO_NA_NO_NORM;
    AERO_REQUIRE(nonorm || p->scope != 1 || (p->groups >= 1 && p->groups <= kNaMaxGroups && p->C % p->groups == 0 && (p->C / p->groups) % 4 == 0),
                 "aero_norm_act_train: groups (group width must be a multiple of 4)");
    AERO_REQUIRE(p->scope == 1 || (p->f_off == 0 && p->F_in == p->F_out), "aero_norm_act_train: crop needs scope 1");
    AERO_REQUIRE(p->f_off >= 0 && p->f_off + p->F_out <= p->F_in, "aero_norm_act_train: crop out of range");
    AERO_REQUIRE(p->op != AERO_NA_SNAKE || p->scope == 2, "aero_norm_act_train: snake needs the per-row scope");
    return AERO_OK;
}

static dim3 na_train_grid(const aero_norm_act_params* p, bool input_rows) {
    const bool glu = (p->op == AERO_NA_GLU || p->op == AERO_NA_GLU_SCALE_RES);
    const int Cout = glu ? p->C / 2 : p->C;
    const int ppp = 256 / (Cout / 4);
    const int rows = input_rows ? p->F_in : p->F_out;
    const int64_t npix = (p->scope == 2) ? (int64_t)p->T : (int64_t)rows * p->T;
    const int nseg = (p->scope == 2) ? p->B * p->F_in : p->B;
    int chunks = (int)((npix + (int64_t)ppp * 8 - 1) / ((int64_t)ppp * 8));
    if (chunks < 1) chunks = 1;
    return dim3((unsigned)chunks, (unsigned)nseg);
}

extern "C" int aero_norm_act_train_fwd(const float* x, const double* stats, const float* gamma, const float* beta, const float* snake_a,
                                       const float* scale, const float* residual, float* y, const aero_norm_act_params* p,
                                       aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && y && p, "aero_norm_act_train_fwd: null argument");
    int rc = na_train_check(p);
    if (rc != AERO_OK) return rc;
    AERO_REQUIRE((p->flags & AERO_NA_NO_NORM) || (stats && gamma && beta), "aero_norm_act_train_fwd: statistics / affine missing");
    const dim3 grid = na_train_grid(p, false);
    AERO_REQUIRE(grid.y <= 65535, "aero_norm_act_train_fwd: too many segments");
    cudaStream_t st = (cudaStream_t)stream;
#define AERO_NAT(OP) na_train_fwd_kernel<OP><<<grid, 256, 0, st>>>(x, stats, gamma, beta, snake_a, scale, residual, y, *p)
    switch (p->op) {
        case AERO_NA_NONE: AERO_NAT(AERO_NA_NONE); break;
        case AERO_NA_GELU: AERO_NAT(AERO_NA_GELU); break;
        case AERO_NA_GLU: AERO_NAT(AERO_NA_GLU); break;
        case AERO_NA_SNAKE: AERO_NAT(AERO_NA_SNAKE); break;
        case AERO_NA_GLU_SCALE_RES: AERO_NAT(AERO_NA_GLU_SCALE_RES); break;
        case AERO_NA_RELU: AERO_NAT(AERO_NA_RELU); break;
        case AERO_NA_LEAKY: AERO_NAT(AERO_NA_LEAKY); break;
        case AERO_NA_TANH: AERO_NAT(AERO_NA_TANH); break;
        default: set_error("aero_norm_act_train_fwd: op=%d", p->op); return AERO_ERR_INVALID;
    }
#undef AERO_NAT
    return check_launch("aero_norm_act_train_fwd");
}

extern "C" int aero_norm_act_train_bwd(const float* x, const double* stats, const float* gamma, const float* beta, const float* snake_a,
                                       const float* scale, const float* dy, float* dx, double* dgamma, double* dbeta, double* dscale,
                                       double* dsnake, double* ws, int32_t pass, const aero_norm_act_params* p, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && dy && p && (pass == 1 || pass == 2), "aero_norm_act_train_bwd: null argument");
    int rc = na_train_check(p);
    if (rc != AERO_OK) return rc;
    const bool nonorm = p->flags & AERO_NA_NO_NORM;
    AERO_REQUIRE(nonorm || (stats && gamma && beta && dgamma && dbeta && (p->scope == 3 || ws)), "aero_norm_act_train_bwd: missing buffers");
    AERO_REQUIRE(pass == 1 || dx, "aero_norm_act_train_bwd: dx missing");
    const dim3 grid = na_train_grid(p, true);
    AERO_REQUIRE(grid.y <= 65535, "aero_norm_act_train_bwd: too many segments");
    cudaStream_t st = (cudaStream_t)stream;
#define AERO_NAB(OP)                                                                                                                    \
    if (pass == 1) na_train_bwd_kernel<OP, false><<<grid, 256, 0, st>>>(x, stats, gamma, beta, snake_a, scale, dy, dx, dgamma, dbeta, dscale, dsnake, ws, *p); \
    else na_train_bwd_kernel<OP, true><<<grid, 256, 0, st>>>(x, stats, gamma, beta, snake_a, scale, dy, dx, dgamma, dbeta, dscale, dsnake, ws, *p)
    switch (p->op) {
        case AERO_NA_NONE: AERO_NAB(AERO_NA_NONE); break;
        case AERO_NA_GELU: AERO_NAB(AERO_NA_GELU); break;
        case AERO_NA_GLU: AERO_NAB(AERO_NA_GLU); break;
        case AERO_NA_SNAKE: AERO_NAB(AERO_NA_SNAKE); break;
        case AERO_NA_GLU_SCALE_RES: AERO_NAB(AERO_NA_GLU_SCALE_RES); break;
        case AERO_NA_RELU: AERO_NAB(AERO_NA_RELU); break;
        case AERO_NA_LEAKY: AERO_NAB(AERO_NA_LEAKY); break;
        case AERO_NA_TANH: AERO_NAB(AERO_NA_TANH); break;
        default: set_error("aero_norm_act_train_bwd: op=%d", p->op); return AERO_ERR_INVALID;
    }
#undef AERO_NAB
    return check_launch("aero_norm_act_train_bwd");
}

extern "C" int aero_adam_step(const void* chunk_table, int32_t n_chunks, float lr, float beta1, float beta2, float eps, int32_t step,
                              float grad_scale, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(chunk_table && n_chunks >= 1 && step >= 1, "aero_adam_step: bad argument");
    const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    adam_kernel<<<(unsigned)n_chunks, 256, 0, (cudaStream_t)stream>>>(static_cast<const AdamChunk*>(chunk_table), lr, beta1, beta2, eps, (float)bc1,
                                                                     (float)sqrt(bc2), grad_scale);
    return check_launch("aero_adam_step");
}
