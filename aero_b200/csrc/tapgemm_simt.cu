// Tap-GEMM, fp32 SIMT implementation (exact-fp32 accumulate; the parity anchor and the fallback
// for shapes the wgmma path does not take).  See include/aero_b200.h for the operator contract.
//
// Tile: BM pixels (consecutive t inside one (b, f_out) row) x BN output columns, K consumed in
// chunks of 16 channels per tap; 256 threads, TM x TN register tile per thread.
#include "tapgemm.cuh"

namespace aero {

constexpr int kBK = 16;


template <int BM, int BN, int TM, int TN, typename TA, typename TO>
__global__ void __launch_bounds__((BM / TM) * (BN / TN)) tapgemm_simt_kernel(const TapGemmArgs g) {
    constexpr int NT = (BM / TM) * (BN / TN);
    constexpr int TX = BN / TN;
    static_assert(NT == 256, "tile shape must give 256 threads");
    __shared__ __align__(16) float As[kBK][BM + 4];
    __shared__ __align__(16) float Bs[kBK][BN + 4];
    __shared__ double sred[NT / 32][8][2];

    const aero_tapgemm_params& p = g.p;
    const int tid = threadIdx.x;
    const int tx = tid % TX, ty = tid / TX;
    const int tile = blockIdx.x;
    const int tt = tile % g.tiles_t;
    const int row = tile / g.tiles_t;
    const int fo = row % p.F_out;
    const int b = row / p.F_out;
    const int t0 = tt * BM;
    const int n0 = blockIdx.y * BN;
    const int K = p.C1 + p.C2;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    const float* wb = static_cast<const float*>(g.w) + (int64_t)b * p.w_sb;
    const TA* const ga1 = static_cast<const TA*>(g.a1);
    const TA* const ga2 = static_cast<const TA*>(g.a2);

    for (int tap = 0; tap < g.ntaps; ++tap) {
        int fi, dt, slab;
        if (p.mode == AERO_TAPS_CONV) {
            const int jf = tap / p.kt, jt = tap - jf * p.kt;
            fi = fo * p.stride_f + jf - p.pad_f;
            dt = jt * p.dil_t - p.pad_t;
            slab = tap;
        } else {
            const int fof = fo + p.f_out_offset;
            const int kidx = fof % p.stride_f + tap * p.stride_f;
            fi = fof / p.stride_f - tap;
            dt = 0;
            slab = kidx;
        }
        if (fi < 0 || fi >= p.F_in) continue;          // uniform across the CTA
        const TA* s1 = ga1 ? ga1 + (int64_t)b * p.a1_sb + (int64_t)fi * p.a1_sf : nullptr;
        const TA* s2 = ga2 ? ga2 + (int64_t)b * p.a2_sb + (int64_t)fi * p.a2_sf : nullptr;
        const float* wslab = wb + (int64_t)slab * K * g.ldw;

        for (int kc = 0; kc < K; kc += kBK) {
            // ---- A tile: BM x 16, thread loads 4 consecutive channels of (BM*16/4)/256 pixels
#pragma unroll
            for (int it = 0; it < (BM * kBK / 4) / NT; ++it) {
                const int e = tid + it * NT;
                const int m = e >> 2, c4 = (e & 3) * 4;
                const int ti = t0 + m + dt;
                const int c = kc + c4;
                float v[4] = {0.f, 0.f, 0.f, 0.f};
                if (ti >= 0 && ti < p.T_in && (t0 + m) < p.T) {
                    if (g.vec_a && c + 3 < p.C1) {
                        const float4 q = ld4(s1 + (int64_t)ti * p.a1_st + c);
                        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
                    } else if (g.vec_a && c >= p.C1 && c + 3 < K) {
                        const float4 q = ld4(s2 + (int64_t)ti * p.a2_st + (c - p.C1));
                        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
                    } else {
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            const int cc = c + u;
                            if (cc < p.C1) v[u] = ldf(s1 + (int64_t)ti * p.a1_st + cc);
                            else if (cc < K) v[u] = ldf(s2 + (int64_t)ti * p.a2_st + (cc - p.C1));
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) As[c4 + u][m] = v[u];
            }
            // ---- W tile: 16 x BN
#pragma unroll
            for (int it = 0; it < (kBK * BN / 4 + NT - 1) / NT; ++it) {
                const int e = tid + it * NT;
                if (e < kBK * BN / 4) {
                    const int kk = e / (BN / 4), n4 = (e % (BN / 4)) * 4;
                    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (kc + kk < K && n0 + n4 < g.ldw)
                        q = *reinterpret_cast<const float4*>(wslab + (int64_t)(kc + kk) * g.ldw + n0 + n4);
                    *reinterpret_cast<float4*>(&Bs[kk][n4]) = q;
                }
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < kBK; ++kk) {
                float a[TM], bb[TN];
#pragma unroll
                for (int i = 0; i < TM; i += 4) {
                    const float4 q = *reinterpret_cast<const float4*>(&As[kk][ty * TM + i]);
                    a[i] = q.x; a[i + 1] = q.y; a[i + 2] = q.z; a[i + 3] = q.w;
                }
                if (TN >= 4) {
#pragma unroll
                    for (int j = 0; j < TN; j += 4) {
                        const float4 q = *reinterpret_cast<const float4*>(&Bs[kk][tx * TN + j]);
                        bb[j] = q.x; bb[j + 1] = q.y; bb[j + 2] = q.z; bb[j + 3] = q.w;
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < TN; ++j) bb[j] = Bs[kk][tx * TN + j];
                }
#pragma unroll
                for (int i = 0; i < TM; ++i)
#pragma unroll
                    for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
            }
            __syncthreads();
        }
    }

    // ------------------------------------------------------------------ epilogue
    const int Nout = p.glu ? p.N / 2 : p.N;
    constexpr int TNO_MAX = TN;
    float ssum = 0.f, ssq = 0.f;
    const int gw = (p.stats_mode == 1) ? Nout / p.groups : Nout;
    float sa = 1.f, sb = 0.f;
    if (g.samp_affine) { sa = g.samp_affine[2 * b]; sb = g.samp_affine[2 * b + 1]; }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int t = t0 + ty * TM + i;
        if (t >= p.T) continue;
        float v[TN];
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + tx * TN + j;
            float x = acc[i][j];
            if (n < p.N) {
                if (g.bias) x += g.bias[n];
                if (g.colscale) x *= g.colscale[(int64_t)b * p.cs_sb + (int64_t)t * p.cs_st + n];
                if (p.act == AERO_ACT_GELU) x = gelu_exact(x);
                else if (p.act == AERO_ACT_RELU) x = fmaxf(x, 0.f);
                else if (p.act == AERO_ACT_LEAKY) x = leaky_f(x);
                else if (p.act == AERO_ACT_TANH) x = tanhf(x);
            }
            v[j] = x;
        }
        float o[TNO_MAX];
        int no0, cnt;
        if (p.glu) {
            // TN is even whenever glu is requested (host checks): pairs (2j, 2j+1)
            no0 = (n0 + tx * TN) >> 1;
            cnt = TN / 2;
#pragma unroll
            for (int j = 0; j < TN / 2; ++j) o[j] = v[2 * j] * sigmoid_f(v[2 * j + 1]);
        } else {
            no0 = n0 + tx * TN;
            cnt = TN;
#pragma unroll
            for (int j = 0; j < TN; ++j) o[j] = v[j];
        }
        TO* op = static_cast<TO*>(g.out) + (int64_t)b * p.o_sb + (int64_t)fo * p.o_sf + (int64_t)t * p.o_st;
        const TO* rp = g.residual ? static_cast<const TO*>(g.residual) + (int64_t)b * p.r_sb + (int64_t)fo * p.r_sf + (int64_t)t * p.r_st : nullptr;
#pragma unroll
        for (int j = 0; j < TNO_MAX; ++j) {
            if (j < cnt && no0 + j < Nout) {
                float x = o[j];
                if (g.addend_fn) x += g.addend_fn[(int64_t)fo * Nout + no0 + j];
                if (rp) x += ldf(rp + no0 + j);
                x = x * sa + sb;
                if ((p.flags & 1) && sizeof(TO) == 4) x = round_tf32_rna(x);
                x = stored(x, op);
                o[j] = x;
                ssum += x;
                ssq += x * x;
            }
        }
        if (g.vec_o && !p.glu && TN == 4 && no0 + 3 < Nout) {
            st4(op + no0, make_float4(o[0], o[1], o[2], o[3]));
        } else {
#pragma unroll
            for (int j = 0; j < TNO_MAX; ++j)
                if (j < cnt && no0 + j < Nout) stf(op + no0 + j, o[j]);
        }
    }

    if (p.stats_mode != 0 && g.stats != nullptr) {
        // all columns of a thread fall in one group (host guarantees gw % TN' == 0)
        const int no_first = p.glu ? (n0 + tx * TN) >> 1 : n0 + tx * TN;
        const int my_g = no_first < Nout ? no_first / gw : -1;
        const int g_lo = (p.glu ? n0 >> 1 : n0) / gw;
        const int warp = tid >> 5, lane = tid & 31;
#pragma unroll 1
        for (int q = 0; q < 8; ++q) {
            const float s = (my_g == g_lo + q) ? ssum : 0.f;
            const float s2 = (my_g == g_lo + q) ? ssq : 0.f;
            const double ds = warp_sum((double)s), dq = warp_sum((double)s2);
            if (lane == 0) { sred[warp][q][0] = ds; sred[warp][q][1] = dq; }
        }
        __syncthreads();
        if (tid < 8) {
            double a = 0, c = 0;
            for (int w = 0; w < NT / 32; ++w) { a += sred[w][tid][0]; c += sred[w][tid][1]; }
            const int gi = g_lo + tid;
            const int ngroups = (p.stats_mode == 1) ? p.groups : 1;
            if (gi < ngroups && (a != 0.0 || c != 0.0)) {
                const int64_t slot = (p.stats_mode == 1) ? ((int64_t)b * p.groups + gi) : ((int64_t)b * p.F_out + fo);
                atomicAdd(&g.stats[2 * slot], a);
                atomicAdd(&g.stats[2 * slot + 1], c);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Thin shapes are HBM-bound, not FLOP-bound; the tiled kernel above wastes most of its tile on them.
//
// thin-N (N <= 8: FTB's C->5 squeeze, the final 96->2 transposed conv): one thread per output pixel computes all N
// columns over all taps; the weights live in shared memory ([tap][c][8]) and are read as broadcasts.
constexpr int kThinN = 8;

template <typename TA, typename TO>
__global__ void __launch_bounds__(256) tapgemm_thin_n_kernel(const TapGemmArgs g) {
    extern __shared__ __align__(16) float wsm[];          // [nslab][K][8]
    const aero_tapgemm_params& p = g.p;
    const int K = p.C1 + p.C2;
    const int nslab = (p.mode == AERO_TAPS_CONVT) ? p.kf : p.kf * p.kt;
    for (int i = threadIdx.x; i < nslab * K * kThinN; i += blockDim.x) {
        const int n = i % kThinN, rk = i / kThinN;
        wsm[i] = n < p.N ? static_cast<const float*>(g.w)[(int64_t)rk * g.ldw + n] : 0.f;
    }
    __syncthreads();
    const int64_t npix = (int64_t)p.B * p.F_out * p.T;
    PixelWalk pw;
    pw.init((int64_t)blockIdx.x * blockDim.x + threadIdx.x, (int64_t)gridDim.x * blockDim.x, p.T, p.F_out);
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += (int64_t)gridDim.x * blockDim.x, pw.next()) {
        const int t = pw.t, fo = pw.f, b = pw.b;
        float acc[kThinN];
#pragma unroll
        for (int n = 0; n < kThinN; ++n) acc[n] = 0.f;
        for (int tap = 0; tap < g.ntaps; ++tap) {
            int fi, dt, slab;
            if (p.mode == AERO_TAPS_CONV) {
                const int jf = tap / p.kt, jt = tap - jf * p.kt;
                fi = fo * p.stride_f + jf - p.pad_f; dt = jt * p.dil_t - p.pad_t; slab = tap;
            } else {
                const int fof = fo + p.f_out_offset;
                fi = fof / p.stride_f - tap; dt = 0; slab = fof % p.stride_f + tap * p.stride_f;
            }
            const int ti = t + dt;
            if (fi < 0 || fi >= p.F_in || ti < 0 || ti >= p.T_in) continue;
            const float* wt = wsm + (int64_t)slab * K * kThinN;
            for (int src = 0; src < 2; ++src) {
                const int Cs = src ? p.C2 : p.C1;
                if (Cs == 0) continue;
                const TA* a = src ? static_cast<const TA*>(g.a2) + (int64_t)b * p.a2_sb + (int64_t)fi * p.a2_sf + (int64_t)ti * p.a2_st
                                  : static_cast<const TA*>(g.a1) + (int64_t)b * p.a1_sb + (int64_t)fi * p.a1_sf + (int64_t)ti * p.a1_st;
                const float* wc = wt + (src ? p.C1 : 0) * kThinN;
                for (int c = 0; c < Cs; c += 4) {
                    const float4 av = ld4(a + c);       // vec_a holds (host check)
                    const float avs[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const float4 w0 = *reinterpret_cast<const float4*>(wc + (c + u) * kThinN);
                        const float4 w1 = *reinterpret_cast<const float4*>(wc + (c + u) * kThinN + 4);
                        acc[0] = fmaf(avs[u], w0.x, acc[0]); acc[1] = fmaf(avs[u], w0.y, acc[1]);
                        acc[2] = fmaf(avs[u], w0.z, acc[2]); acc[3] = fmaf(avs[u], w0.w, acc[3]);
                        acc[4] = fmaf(avs[u], w1.x, acc[4]); acc[5] = fmaf(avs[u], w1.y, acc[5]);
                        acc[6] = fmaf(avs[u], w1.z, acc[6]); acc[7] = fmaf(avs[u], w1.w, acc[7]);
                    }
                }
            }
        }
        float sa = 1.f, sb = 0.f;
        if (g.samp_affine) { sa = g.samp_affine[2 * b]; sb = g.samp_affine[2 * b + 1]; }
        TO* op = static_cast<TO*>(g.out) + (int64_t)b * p.o_sb + (int64_t)fo * p.o_sf + (int64_t)t * p.o_st;
        const TO* rp = g.residual ? static_cast<const TO*>(g.residual) + (int64_t)b * p.r_sb + (int64_t)fo * p.r_sf + (int64_t)t * p.r_st : nullptr;
#pragma unroll
        for (int n = 0; n < kThinN; ++n) {
            if (n < p.N) {
                float x = acc[n] + (g.bias ? g.bias[n] : 0.f);
                if (p.act == AERO_ACT_GELU) x = gelu_exact(x);
                else if (p.act == AERO_ACT_RELU) x = fmaxf(x, 0.f);
                else if (p.act == AERO_ACT_LEAKY) x = leaky_f(x);
                else if (p.act == AERO_ACT_TANH) x = tanhf(x);
                if (rp) x += ldf(rp + n);
                x = x * sa + sb;
                if ((p.flags & 1) && sizeof(TO) == 4) x = round_tf32_rna(x);
                stf(op + n, x);
            }
        }
    }
}

// thin-N over a long K with few pixels (the discriminator's 1024 -> 1 output layer: 3072-term dot products for a thousand pixels): one
// WARP per pixel, lanes stride the channels, weights straight from L2 (coalesced float4s), shuffle reduction.
template <typename TA, typename TO>
__global__ void __launch_bounds__(256) tapgemm_thin_n_warp_kernel(const TapGemmArgs g) {
    const aero_tapgemm_params& p = g.p;
    const int K = p.C1 + p.C2;
    const int lane = threadIdx.x & 31;
    const int64_t npix = (int64_t)p.B * p.F_out * p.T;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const float* W = static_cast<const float*>(g.w);
    const bool wide = g.ldw > 4;
    for (int64_t pix = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pix < npix; pix += nwarps) {
        const int t = (int)(pix % p.T);
        const int64_t row = pix / p.T;
        const int fo = (int)(row % p.F_out), b = (int)(row / p.F_out);
        float acc[kThinN];
#pragma unroll
        for (int n = 0; n < kThinN; ++n) acc[n] = 0.f;
        for (int tap = 0; tap < g.ntaps; ++tap) {
            int fi, dt, slab;
            if (p.mode == AERO_TAPS_CONV) {
                const int jf = tap / p.kt, jt = tap - jf * p.kt;
                fi = fo * p.stride_f + jf - p.pad_f; dt = jt * p.dil_t - p.pad_t; slab = tap;
            } else {
                const int fof = fo + p.f_out_offset;
                fi = fof / p.stride_f - tap; dt = 0; slab = fof % p.stride_f + tap * p.stride_f;
            }
            const int ti = t + dt;
            if (fi < 0 || fi >= p.F_in || ti < 0 || ti >= p.T_in) continue;
            for (int src = 0; src < 2; ++src) {
                const int Cs = src ? p.C2 : p.C1;
                if (Cs == 0) continue;
                const TA* a = src ? static_cast<const TA*>(g.a2) + (int64_t)b * p.a2_sb + (int64_t)fi * p.a2_sf + (int64_t)ti * p.a2_st
                                  : static_cast<const TA*>(g.a1) + (int64_t)b * p.a1_sb + (int64_t)fi * p.a1_sf + (int64_t)ti * p.a1_st;
                const float* wc = W + ((int64_t)slab * K + (src ? p.C1 : 0)) * g.ldw;
                for (int c = lane * 4; c < Cs; c += 128) {
                    const float4 av = ld4(a + c);
                    const float avs[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const float4 w0 = *reinterpret_cast<const float4*>(wc + (int64_t)(c + u) * g.ldw);
                        acc[0] = fmaf(avs[u], w0.x, acc[0]); acc[1] = fmaf(avs[u], w0.y, acc[1]);
                        acc[2] = fmaf(avs[u], w0.z, acc[2]); acc[3] = fmaf(avs[u], w0.w, acc[3]);
                        if (wide) {
                            const float4 w1 = *reinterpret_cast<const float4*>(wc + (int64_t)(c + u) * g.ldw + 4);
                            acc[4] = fmaf(avs[u], w1.x, acc[4]); acc[5] = fmaf(avs[u], w1.y, acc[5]);
                            acc[6] = fmaf(avs[u], w1.z, acc[6]); acc[7] = fmaf(avs[u], w1.w, acc[7]);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int n = 0; n < kThinN; ++n) acc[n] = warp_sum(acc[n]);
        if (lane != 0) continue;
        float sa = 1.f, sb = 0.f;
        if (g.samp_affine) { sa = g.samp_affine[2 * b]; sb = g.samp_affine[2 * b + 1]; }
        TO* op = static_cast<TO*>(g.out) + (int64_t)b * p.o_sb + (int64_t)fo * p.o_sf + (int64_t)t * p.o_st;
        const TO* rp = g.residual ? static_cast<const TO*>(g.residual) + (int64_t)b * p.r_sb + (int64_t)fo * p.r_sf + (int64_t)t * p.r_st : nullptr;
#pragma unroll
        for (int n = 0; n < kThinN; ++n) {
            if (n < p.N) {
                float x = acc[n] + (g.bias ? g.bias[n] : 0.f);
                if (p.act == AERO_ACT_GELU) x = gelu_exact(x);
                else if (p.act == AERO_ACT_RELU) x = fmaxf(x, 0.f);
                else if (p.act == AERO_ACT_LEAKY) x = leaky_f(x);
                else if (p.act == AERO_ACT_TANH) x = tanhf(x);
                if (rp) x += ldf(rp + n);
                x = x * sa + sb;
                if ((p.flags & 1) && sizeof(TO) == 4) x = round_tf32_rna(x);
                stf(op + n, x);
            }
        }
    }
}

// thin-K (K <= 4, single tap: pre_conv 2->48): a thread owns one quad of output columns (its weights and bias stay in
// registers) and walks over pixels; consecutive lanes = consecutive column quads of one pixel -> 16-byte coalesced stores.
template <typename TA, typename TO>
__global__ void __launch_bounds__(256) tapgemm_thin_k_kernel(const TapGemmArgs g) {
    const aero_tapgemm_params& p = g.p;
    const int K = p.C1;
    const int n4 = p.N >> 2;
    const int ppp = 256 / n4;                             // pixels per pass (host guarantees n4 <= 256)
    const int nq = threadIdx.x % n4, dp = threadIdx.x / n4;
    if (dp >= ppp) return;
    const int n = nq * 4;
    float4 w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = k < K ? *reinterpret_cast<const float4*>(static_cast<const float*>(g.w) + (int64_t)k * g.ldw + n) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 bias = g.bias ? *reinterpret_cast<const float4*>(g.bias + n) : make_float4(0.f, 0.f, 0.f, 0.f);
    const bool rnd = (p.flags & 1) && sizeof(TO) == 4;
    const int64_t npix = (int64_t)p.B * p.F_out * p.T;
    PixelWalk pw;
    pw.init((int64_t)blockIdx.x * ppp + dp, (int64_t)gridDim.x * ppp, p.T, p.F_out);
    for (int64_t pix = (int64_t)blockIdx.x * ppp + dp; pix < npix; pix += (int64_t)gridDim.x * ppp, pw.next()) {
        const int t = pw.t, fo = pw.f, b = pw.b;
        const TA* a = static_cast<const TA*>(g.a1) + (int64_t)b * p.a1_sb + (int64_t)fo * p.a1_sf + (int64_t)t * p.a1_st;
        float4 acc = bias;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (k < K) {
                const float av = ldf(a + k);
                acc.x = fmaf(av, w[k].x, acc.x); acc.y = fmaf(av, w[k].y, acc.y); acc.z = fmaf(av, w[k].z, acc.z); acc.w = fmaf(av, w[k].w, acc.w);
            }
        }
        if (p.act == AERO_ACT_GELU) { acc.x = gelu_exact(acc.x); acc.y = gelu_exact(acc.y); acc.z = gelu_exact(acc.z); acc.w = gelu_exact(acc.w); }
        else if (p.act == AERO_ACT_RELU) { acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f); }
        else if (p.act == AERO_ACT_LEAKY) { acc.x = leaky_f(acc.x); acc.y = leaky_f(acc.y); acc.z = leaky_f(acc.z); acc.w = leaky_f(acc.w); }
        else if (p.act == AERO_ACT_TANH) { acc.x = tanhf(acc.x); acc.y = tanhf(acc.y); acc.z = tanhf(acc.z); acc.w = tanhf(acc.w); }
        if (rnd) { acc.x = round_tf32_rna(acc.x); acc.y = round_tf32_rna(acc.y); acc.z = round_tf32_rna(acc.z); acc.w = round_tf32_rna(acc.w); }
        st4(static_cast<TO*>(g.out) + (int64_t)b * p.o_sb + (int64_t)fo * p.o_sf + (int64_t)t * p.o_st + n, acc);
    }
}

// thin transposed conv (stride_f * N <= 8: the final 96 -> 2 layer, reference aero.py:179,209): the s output rows fed by one
// input row pair are computed together.  With a = fo' / s the taps are fi = a - j, slab = r + j*s for output row
// fo' = a*s + r: treat (r, n) as 8 "virtual columns" of a plain conv over j.  Every input row is then read k/s times
// instead of k times, and each thread keeps all its accumulators.
template <typename TA, typename TO>
__global__ void __launch_bounds__(256) tapgemm_thin_convt_kernel(const TapGemmArgs g, const int a_lo, const int n_a) {
    extern __shared__ __align__(16) float wsm[];          // [ntaps][K][8]: column v = r*N + n
    const aero_tapgemm_params& p = g.p;
    const int K = p.C1, s = p.stride_f, ntaps = p.kf / s;
    for (int i = threadIdx.x; i < ntaps * K * kThinN; i += blockDim.x) {
        const int v = i % kThinN, c = (i / kThinN) % K, j = i / (kThinN * K);
        const int r = v / p.N, n = v % p.N;
        wsm[i] = (r < s) ? static_cast<const float*>(g.w)[((int64_t)(r + j * s) * K + c) * g.ldw + n] : 0.f;
    }
    __syncthreads();
    const int64_t npix = (int64_t)p.B * n_a * p.T;
    PixelWalk pw;
    pw.init((int64_t)blockIdx.x * blockDim.x + threadIdx.x, (int64_t)gridDim.x * blockDim.x, p.T, n_a);
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += (int64_t)gridDim.x * blockDim.x, pw.next()) {
        const int t = pw.t, a = a_lo + pw.f, b = pw.b;
        float acc[kThinN];
#pragma unroll
        for (int v = 0; v < kThinN; ++v) acc[v] = 0.f;
        for (int j = 0; j < ntaps; ++j) {
            const int fi = a - j;
            if (fi < 0 || fi >= p.F_in) continue;
            const TA* src = static_cast<const TA*>(g.a1) + (int64_t)b * p.a1_sb + (int64_t)fi * p.a1_sf + (int64_t)t * p.a1_st;
            const float* wt = wsm + (int64_t)j * K * kThinN;
            for (int c = 0; c < K; c += 4) {
                const float4 av = ld4(src + c);
                const float avs[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float4 w0 = *reinterpret_cast<const float4*>(wt + (c + u) * kThinN);
                    const float4 w1 = *reinterpret_cast<const float4*>(wt + (c + u) * kThinN + 4);
                    acc[0] = fmaf(avs[u], w0.x, acc[0]); acc[1] = fmaf(avs[u], w0.y, acc[1]);
                    acc[2] = fmaf(avs[u], w0.z, acc[2]); acc[3] = fmaf(avs[u], w0.w, acc[3]);
                    acc[4] = fmaf(avs[u], w1.x, acc[4]); acc[5] = fmaf(avs[u], w1.y, acc[5]);
                    acc[6] = fmaf(avs[u], w1.z, acc[6]); acc[7] = fmaf(avs[u], w1.w, acc[7]);
                }
            }
        }
        float sa = 1.f, sb = 0.f;
        if (g.samp_affine) { sa = g.samp_affine[2 * b]; sb = g.samp_affine[2 * b + 1]; }
#pragma unroll
        for (int v = 0; v < kThinN; ++v) {
            const int r = v / p.N, n = v % p.N;
            const int fo = a * s + r - p.f_out_offset;
            if (r < s && fo >= 0 && fo < p.F_out) {
                float x = acc[v] + (g.bias ? g.bias[n] : 0.f);
                if (p.act == AERO_ACT_GELU) x = gelu_exact(x);
                else if (p.act == AERO_ACT_RELU) x = fmaxf(x, 0.f);
                else if (p.act == AERO_ACT_LEAKY) x = leaky_f(x);
                else if (p.act == AERO_ACT_TANH) x = tanhf(x);
                x = x * sa + sb;
                if ((p.flags & 1) && sizeof(TO) == 4) x = round_tf32_rna(x);
                stf(static_cast<TO*>(g.out) + (int64_t)b * p.o_sb + (int64_t)fo * p.o_sf + (int64_t)t * p.o_st + n, x);
            }
        }
    }
}

template <typename TA, typename TO>
static int tapgemm_simt_launch_t(const TapGemmArgs& g, cudaStream_t st) {
    const aero_tapgemm_params& p = g.p;
    TapGemmArgs a = g;
    const bool plain = !p.glu && p.stats_mode == 0 && !g.addend_fn && !g.colscale && p.w_sb == 0;
    const int nslab = (p.mode == AERO_TAPS_CONVT) ? p.kf : p.kf * p.kt;
    if (plain && p.mode == AERO_TAPS_CONVT && p.stride_f * p.N <= kThinN && p.C2 == 0 && g.vec_a && !g.residual &&
        (size_t)(p.kf / p.stride_f) * p.C1 * kThinN * 4 <= 96 * 1024) {
        const size_t smem = (size_t)(p.kf / p.stride_f) * p.C1 * kThinN * 4;
        cudaFuncSetAttribute(tapgemm_thin_convt_kernel<TA, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        const int a_lo = p.f_out_offset / p.stride_f, a_hi = (p.f_out_offset + p.F_out - 1) / p.stride_f;
        const int n_a = a_hi - a_lo + 1;
        const int64_t npix = (int64_t)p.B * n_a * p.T;
        int blocks = (int)((npix + 255) / 256);
        if (blocks > 132 * 16) blocks = 132 * 16;
        tapgemm_thin_convt_kernel<TA, TO><<<blocks, 256, smem, st>>>(a, a_lo, n_a);
        return check_launch("aero_tapgemm_fwd(thin-convt)");
    }
    if (plain && p.N <= kThinN && g.vec_a && (int64_t)nslab * (p.C1 + p.C2) >= 1024 && (int64_t)p.B * p.F_out * p.T <= 132 * 64) {
        const int64_t npix = (int64_t)p.B * p.F_out * p.T;           // long dot products, few pixels: a warp per pixel
        tapgemm_thin_n_warp_kernel<TA, TO><<<(unsigned)cdiv(npix, (int64_t)8), 256, 0, st>>>(a);
        return check_launch("aero_tapgemm_fwd(thin-n, warp per pixel)");
    }
    if (plain && p.N <= kThinN && g.vec_a && (size_t)nslab * (p.C1 + p.C2) * kThinN * 4 <= 96 * 1024) {
        const size_t smem = (size_t)nslab * (p.C1 + p.C2) * kThinN * 4;
        cudaFuncSetAttribute(tapgemm_thin_n_kernel<TA, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        const int64_t npix = (int64_t)p.B * p.F_out * p.T;
        int blocks = (int)((npix + 255) / 256);
        if (blocks > 132 * 16) blocks = 132 * 16;
        tapgemm_thin_n_kernel<TA, TO><<<blocks, 256, smem, st>>>(a);
        return check_launch("aero_tapgemm_fwd(thin-n)");
    }
    if (plain && p.mode == AERO_TAPS_CONV && p.kf == 1 && p.kt == 1 && p.stride_f == 1 && p.pad_f == 0 && p.C2 == 0 && p.C1 <= 4 &&
        p.N % 4 == 0 && p.N <= 1024 && g.vec_o && !g.residual && !g.samp_affine && p.F_in == p.F_out) {
        const int ppp = 256 / (p.N / 4);
        const int64_t npix = (int64_t)p.B * p.F_out * p.T;
        int blocks = (int)((npix + (int64_t)ppp * 8 - 1) / ((int64_t)ppp * 8));
        if (blocks > 132 * 32) blocks = 132 * 32;
        if (blocks < 1) blocks = 1;
        tapgemm_thin_k_kernel<TA, TO><<<blocks, 256, 0, st>>>(a);
        return check_launch("aero_tapgemm_fwd(thin-k)");
    }
    const bool thin = p.N <= 16;
    const int BM = 128;
    a.tiles_t = cdiv(p.T, BM);
    const int64_t tiles = (int64_t)p.B * p.F_out * a.tiles_t;
    if (tiles > 2147483647LL) { set_error("aero_tapgemm_fwd: too many tiles"); return AERO_ERR_INVALID; }
    if (thin) {
        dim3 grid((unsigned)tiles, cdiv(p.N, 16));
        tapgemm_simt_kernel<128, 16, 8, 1, TA, TO><<<grid, 256, 0, st>>>(a);
    } else {
        dim3 grid((unsigned)tiles, cdiv(p.N, 64));
        tapgemm_simt_kernel<128, 64, 8, 4, TA, TO><<<grid, 256, 0, st>>>(a);
    }
    return check_launch("aero_tapgemm_fwd(simt)");
}

int tapgemm_simt_launch(const TapGemmArgs& g, cudaStream_t st) {
    const bool a16 = g.p.flags & AERO_TG_A_F16, o16 = g.p.flags & AERO_TG_OUT_F16;
    if (a16) return o16 ? tapgemm_simt_launch_t<__half, __half>(g, st) : tapgemm_simt_launch_t<__half, float>(g, st);
    return o16 ? tapgemm_simt_launch_t<float, __half>(g, st) : tapgemm_simt_launch_t<float, float>(g, st);
}

}  // namespace aero
