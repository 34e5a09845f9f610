// FTB output conv evaluated through a linear (1x1-conv) input -- see include/aero_b200.h, aero_ftb_lin_out_fwd.
//
// In encoder layer 0 the FTB block (reference modules.py:304-325) is fed by `pre_conv`, a 1x1 convolution of the J = 2*C_in
// spectrogram channels (aero.py:89,112).  Everything FTB does before its last ReLU is linear in that input, so the C-channel
// tensors x = pre_conv(z), freq_fc(x * gate) and cat([.., x]) need never exist: with zm = freq_fc applied to z itself,
//   out[b,f,t,n] = relu( sum_j M[b,t][n][j] zm[b,f,t,j] + M[b,t][n][J] s[f] + sum_j V[n][j] z[b,f,t,j] + d[n] )
// where M[b,t] = gate[b,t,:] . Q is a tiny GEMM.  This kernel is that last line: it reads 2J floats per pixel and writes the
// C-channel output once (HBM-bound on the write), instead of three passes over C-channel tensors.
//
// Thread = (frame t, 8 output channels); its 8 x (J+1) slice of M[b,t], V and d stay in registers while it walks down the
// frequency rows.  Consecutive threads write consecutive 16 / 32-byte pieces of one (b, f) row.
#include "common.cuh"

namespace aero {

constexpr int kFtbTT = 32;      // frames per CTA
constexpr int kFtbFS = 8;       // frequency rows are split over gridDim.z CTAs (at most this many)

// Thread = (frame t, 4 output channels); its 4 x (J+1) slice of M[b,t], V and d stay in registers while it walks down its
// share of the frequency rows (two rows per iteration so that four independent loads are in flight).  Consecutive threads
// write consecutive 8 / 16-byte pieces of one (b, f) row.
template <int J, typename TO>
__global__ void __launch_bounds__(512, (J == 2 ? 2 : 1)) ftb_lin_out_kernel(const float* __restrict__ z, const float* __restrict__ zm,
                                                             const float* __restrict__ M, const float* __restrict__ s,
                                                             const float* __restrict__ V, const float* __restrict__ d,
                                                             TO* __restrict__ out, const aero_ftb_lin_params p) {
    const int n4 = p.N >> 2;
    const int tl = threadIdx.x / n4, oc = threadIdx.x - tl * n4;
    const int t = blockIdx.x * kFtbTT + tl, b = blockIdx.y;
    if (t >= p.T) return;
    const int fper = (p.F + gridDim.z - 1) / gridDim.z;
    const int f_lo = blockIdx.z * fper, f_hi = min(p.F, f_lo + fper);
    const int n0 = oc * 4;
    float m[4][J + 1], v[4][J], dd[4];
    const float* Mp = M + ((int64_t)b * p.T + t) * p.N * (J + 1) + (int64_t)n0 * (J + 1);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j <= J; ++j) m[i][j] = Mp[i * (J + 1) + j];
#pragma unroll
        for (int j = 0; j < J; ++j) v[i][j] = V[(n0 + i) * J + j];
        dd[i] = d[n0 + i];
    }
    const float* zp = z + (int64_t)b * p.z_sb + (int64_t)f_lo * p.z_sf + (int64_t)t * J;
    const float* zmp = zm + (int64_t)b * p.zm_sb + (int64_t)f_lo * p.zm_sf + (int64_t)t * J;
    const int64_t ostep = (int64_t)p.T * p.N;
    TO* op = out + (((int64_t)b * p.F + f_lo) * p.T + t) * p.N + n0;
    const bool rnd = sizeof(TO) == 4 && (p.flags & AERO_TG_ROUND_TF32);
    auto row = [&](const float (&a)[J], const float (&am)[J], float sf, TO* dst) {
        float o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float x = fmaf(m[i][J], sf, dd[i]);
#pragma unroll
            for (int j = 0; j < J; ++j) x = fmaf(m[i][j], am[j], fmaf(v[i][j], a[j], x));
            o[i] = fmaxf(x, 0.f);
            if (rnd) o[i] = round_tf32_rna(o[i]);
        }
        st4(dst, make_float4(o[0], o[1], o[2], o[3]));
    };
    int f = f_lo;
    for (; f + 1 < f_hi; f += 2) {
        float a0[J], m0[J], a1[J], m1[J];
#pragma unroll
        for (int j = 0; j < J; j += 2) {
            const float2 q0 = *reinterpret_cast<const float2*>(zp + j), r0 = *reinterpret_cast<const float2*>(zmp + j);
            const float2 q1 = *reinterpret_cast<const float2*>(zp + p.z_sf + j), r1 = *reinterpret_cast<const float2*>(zmp + p.zm_sf + j);
            a0[j] = q0.x; a0[j + 1] = q0.y; m0[j] = r0.x; m0[j + 1] = r0.y;
            a1[j] = q1.x; a1[j + 1] = q1.y; m1[j] = r1.x; m1[j + 1] = r1.y;
        }
        const float s0 = __ldg(s + f), s1 = __ldg(s + f + 1);
        row(a0, m0, s0, op);
        row(a1, m1, s1, op + ostep);
        zp += 2 * p.z_sf; zmp += 2 * p.zm_sf; op += 2 * ostep;
    }
    if (f < f_hi) {
        float a0[J], m0[J];
#pragma unroll
        for (int j = 0; j < J; j += 2) {
            const float2 q0 = *reinterpret_cast<const float2*>(zp + j), r0 = *reinterpret_cast<const float2*>(zmp + j);
            a0[j] = q0.x; a0[j + 1] = q0.y; m0[j] = r0.x; m0[j + 1] = r0.y;
        }
        row(a0, m0, __ldg(s + f), op);
    }
}

// FTB squeeze through the linear pre_conv:  R[b][t][f*r + n] = relu( sum_j W1p[n][j] z[b,f,t,j] + b1p[n] ),  r <= 8.
// z is read along t (its contiguous axis), R is written along f (its contiguous axis): the tile goes through shared memory.
constexpr int kSqT = 32, kSqF = 32;
template <int J, typename TO>
__global__ void __launch_bounds__(256) ftb_lin_squeeze_kernel(const float* __restrict__ z, const float* __restrict__ W1p,
                                                              const float* __restrict__ b1p, TO* __restrict__ R,
                                                              const aero_ftb_lin_params p, const int r) {
    __shared__ float tile[kSqT][kSqF * 8 + 1];
    const int t0 = blockIdx.x * kSqT, f0 = blockIdx.y * kSqF, b = blockIdx.z;
    float w[8][J], bb[8];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
        for (int j = 0; j < J; ++j) w[n][j] = n < r ? W1p[n * J + j] : 0.f;
        bb[n] = n < r ? b1p[n] : 0.f;
    }
    // phase 1: thread = (t fast, f slow): coalesced float2 / float4 reads along t
    for (int i = threadIdx.x; i < kSqT * kSqF; i += 256) {
        const int tl = i % kSqT, fl = i / kSqT;
        const int t = t0 + tl, f = f0 + fl;
        if (t < p.T && f < p.F) {
            const float* zp = z + (int64_t)b * p.z_sb + (int64_t)f * p.z_sf + (int64_t)t * J;
            float a[J];
#pragma unroll
            for (int j = 0; j < J; j += 2) { const float2 q = *reinterpret_cast<const float2*>(zp + j); a[j] = q.x; a[j + 1] = q.y; }
#pragma unroll
            for (int n = 0; n < 8; ++n) {
                if (n < r) {
                    float x = bb[n];
#pragma unroll
                    for (int j = 0; j < J; ++j) x = fmaf(w[n][j], a[j], x);
                    tile[tl][fl * r + n] = fmaxf(x, 0.f);
                }
            }
        }
    }
    __syncthreads();
    // phase 2: each frame's kSqF*r outputs are contiguous in R
    const int cols = min(kSqF, p.F - f0) * r;
    const bool rnd = sizeof(TO) == 4 && (p.flags & AERO_TG_ROUND_TF32);
    for (int i = threadIdx.x; i < kSqT * cols; i += 256) {
        const int tl = i / cols, c = i - tl * cols;
        const int t = t0 + tl;
        if (t < p.T) {
            float x = tile[tl][c];
            if (rnd) x = round_tf32_rna(x);
            stf(R + ((int64_t)b * p.T + t) * ((int64_t)p.F * r) + (int64_t)f0 * r + c, x);
        }
    }
}

}  // namespace aero

extern "C" int aero_ftb_lin_out_fwd(const float* z, const float* zm, const float* M, const float* s, const float* V,
                                    const float* d, void* out, const aero_ftb_lin_params* p, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(z && zm && M && s && V && d && out && p, "aero_ftb_lin_out_fwd: null argument");
    AERO_REQUIRE(p->B >= 1 && p->F >= 1 && p->T >= 1 && p->N >= 8 && p->N % 8 == 0 && p->N <= 64, "aero_ftb_lin_out_fwd: N=%d (multiple of 8, at most 64)", p->N);
    AERO_REQUIRE(p->J == 2 || p->J == 4, "aero_ftb_lin_out_fwd: J=%d (2 or 4 input channels)", p->J);
    AERO_REQUIRE(p->z_sf % 2 == 0 && p->z_sb % 2 == 0 && p->zm_sf % 2 == 0 && p->zm_sb % 2 == 0 &&
                     (((uintptr_t)z | (uintptr_t)zm) & 7) == 0 && ((uintptr_t)out & 15) == 0,
                 "aero_ftb_lin_out_fwd: alignment");
    int fs = kFtbFS;
    while (fs > 1 && p->F / fs < 8) fs >>= 1;
    dim3 grid(cdiv(p->T, kFtbTT), p->B, fs);
    const int threads = kFtbTT * (p->N / 4);
    cudaStream_t st = (cudaStream_t)stream;
    const bool o16 = p->flags & AERO_TG_OUT_F16;
#define AERO_FL(JJ)                                                                                                         \
    if (o16) ftb_lin_out_kernel<JJ, __half><<<grid, threads, 0, st>>>(z, zm, M, s, V, d, static_cast<__half*>(out), *p);     \
    else ftb_lin_out_kernel<JJ, float><<<grid, threads, 0, st>>>(z, zm, M, s, V, d, static_cast<float*>(out), *p)
    if (p->J == 2) { AERO_FL(2); } else { AERO_FL(4); }
#undef AERO_FL
    return check_launch("aero_ftb_lin_out_fwd");
}

extern "C" int aero_ftb_lin_squeeze_fwd(const float* z, const float* W1p, const float* b1p, void* R, int32_t r,
                                        const aero_ftb_lin_params* p, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(z && W1p && b1p && R && p, "aero_ftb_lin_squeeze_fwd: null argument");
    AERO_REQUIRE(r >= 1 && r <= 8 && (p->J == 2 || p->J == 4), "aero_ftb_lin_squeeze_fwd: r=%d J=%d", r, p->J);
    AERO_REQUIRE(p->z_sf % 2 == 0 && p->z_sb % 2 == 0 && ((uintptr_t)z & 7) == 0, "aero_ftb_lin_squeeze_fwd: alignment");
    AERO_REQUIRE(p->B <= 65535 && cdiv(p->F, kSqF) <= 65535, "aero_ftb_lin_squeeze_fwd: grid");
    dim3 grid(cdiv(p->T, kSqT), cdiv(p->F, kSqF), p->B);
    cudaStream_t st = (cudaStream_t)stream;
    const bool o16 = p->flags & AERO_TG_OUT_F16;
#define AERO_SQ(JJ)                                                                                                  \
    if (o16) ftb_lin_squeeze_kernel<JJ, __half><<<grid, 256, 0, st>>>(z, W1p, b1p, static_cast<__half*>(R), *p, r);    \
    else ftb_lin_squeeze_kernel<JJ, float><<<grid, 256, 0, st>>>(z, W1p, b1p, static_cast<float*>(R), *p, r)
    if (p->J == 2) { AERO_SQ(2); } else { AERO_SQ(4); }
#undef AERO_SQ
    return check_launch("aero_ftb_lin_squeeze_fwd");
}

// ------------------------------------------------------------------------------------------------
// FTB frequency mix for the deep layers (F = 8 / 16 rows): out[b][g][m] = gate[b][m] * sum_f W[g][f] * x[b][f][m].
// With so few rows the tensor-core tile (128 pixels x F) is all per-tile overhead (measured 170 us for 98 MB at F = 8);
// here a thread keeps the F inputs of 4 consecutive positions in registers and produces the F outputs: one read and one
// write of the tensor at copy bandwidth.
namespace aero {

template <int F, typename TA, typename TO>
__global__ void __launch_bounds__(256) freq_mix_small_kernel(const TA* __restrict__ x, const float* __restrict__ W,
                                                             const float* __restrict__ gate, TO* __restrict__ out,
                                                             const int64_t M, const int flags) {
    __shared__ float ws[F * F];
    for (int i = threadIdx.x; i < F * F; i += 256) ws[i] = W[i];
    __syncthreads();
    const int b = blockIdx.y;
    const bool rnd = sizeof(TO) == 4 && (flags & AERO_TG_ROUND_TF32);
    const TA* xb = x + (int64_t)b * F * M;
    TO* ob = out + (int64_t)b * F * M;
    for (int64_t m = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 4; m < M; m += (int64_t)gridDim.x * 256 * 4) {
        float4 v[F];
#pragma unroll
        for (int f = 0; f < F; ++f) v[f] = ld4(xb + (int64_t)f * M + m);
        const float4 gt = gate ? *reinterpret_cast<const float4*>(gate + (int64_t)b * M + m) : make_float4(1.f, 1.f, 1.f, 1.f);
#pragma unroll 1                      // (unrolled, the compiler keeps all F*F weights in registers: 255 registers and spills at F = 16)
        for (int g = 0; g < F; ++g) {
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int f = 0; f < F; ++f) {
                const float w = ws[g * F + f];
                a.x = fmaf(w, v[f].x, a.x); a.y = fmaf(w, v[f].y, a.y); a.z = fmaf(w, v[f].z, a.z); a.w = fmaf(w, v[f].w, a.w);
            }
            a.x *= gt.x; a.y *= gt.y; a.z *= gt.z; a.w *= gt.w;
            if (rnd) { a.x = round_tf32_rna(a.x); a.y = round_tf32_rna(a.y); a.z = round_tf32_rna(a.z); a.w = round_tf32_rna(a.w); }
            st4(ob + (int64_t)g * M + m, a);
        }
    }
}

template <int F>
static int freq_mix_small_go(const void* x, const float* W, const float* gate, void* out, int B, int64_t M, int flags, cudaStream_t st) {
    int blocks = (int)((M / 4 + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    dim3 grid(blocks < 1 ? 1 : blocks, B);
    const bool a16 = flags & AERO_TG_A_F16, o16 = flags & AERO_TG_OUT_F16;
    if (a16 && o16) freq_mix_small_kernel<F, __half, __half><<<grid, 256, 0, st>>>((const __half*)x, W, gate, (__half*)out, M, flags);
    else if (!a16 && !o16) freq_mix_small_kernel<F, float, float><<<grid, 256, 0, st>>>((const float*)x, W, gate, (float*)out, M, flags);
    else { set_error("aero_freq_mix_small_fwd: input and output must share a storage type"); return AERO_ERR_UNSUPPORTED; }
    return check_launch("aero_freq_mix_small_fwd");
}

}  // namespace aero

extern "C" int aero_freq_mix_small_fwd(const void* x, const float* W, const float* gate, void* out, int32_t B, int32_t F, int64_t M,
                                       int32_t flags, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && W && out && B >= 1 && B <= 65535 && M >= 4, "aero_freq_mix_small_fwd: bad argument");
    AERO_REQUIRE(M % 4 == 0 && (((uintptr_t)x | (uintptr_t)out | (uintptr_t)gate) & 15) == 0, "aero_freq_mix_small_fwd: M %% 4 and 16-byte alignment");
    cudaStream_t st = (cudaStream_t)stream;
    if (F == 8) return freq_mix_small_go<8>(x, W, gate, out, B, M, flags, st);
    if (F == 16) return freq_mix_small_go<16>(x, W, gate, out, B, M, flags, st);
    set_error("aero_freq_mix_small_fwd: F=%d (8 or 16)", F);
    return AERO_ERR_UNSUPPORTED;
}
