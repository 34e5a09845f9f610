// HBM-bound normalisation / activation passes.  See include/aero_b200.h for contracts.
// All kernels move 16 bytes per thread per access along the contiguous channel axis.
#include "common.cuh"

namespace aero {

// ------------------------------------------------------------------------- sample_norm
// reference aero.py:462-464: mean / unbiased std over (C,F,T); y = (x-mean)/(1e-5+std)
__global__ void __launch_bounds__(256) sample_norm_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                                          float* __restrict__ y, float* __restrict__ samp_affine,
                                                          int64_t count, int64_t per_sample, int rnd) {
    const int b = blockIdx.y;
    __shared__ float s_mean, s_inv;
    if (threadIdx.x == 0) {
        const double n = (double)count;                 // statistics cover `count` values; `per_sample` floats are transformed
        const double mean = stats[2 * b] / n;
        double var = (stats[2 * b + 1] - n * mean * mean) / (n - 1.0);
        if (var < 0) var = 0;
        const double sd = sqrt(var);
        s_mean = (float)mean;
        s_inv = (float)(1.0 / (1e-5 + sd));
        if (blockIdx.x == 0 && samp_affine) {
            samp_affine[2 * b] = (float)sd;
            samp_affine[2 * b + 1] = (float)mean;
        }
    }
    __syncthreads();
    const float mean = s_mean, inv = s_inv;
    const float* xb = x + (int64_t)b * per_sample;
    float* yb = y + (int64_t)b * per_sample;
    const int64_t n4 = per_sample >> 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 v = reinterpret_cast<const float4*>(xb)[i];
        v.x = (v.x - mean) * inv; v.y = (v.y - mean) * inv; v.z = (v.z - mean) * inv; v.w = (v.w - mean) * inv;
        if (rnd) { v.x = round_tf32_rna(v.x); v.y = round_tf32_rna(v.y); v.z = round_tf32_rna(v.z); v.w = round_tf32_rna(v.w); }
        reinterpret_cast<float4*>(yb)[i] = v;
    }
    if (blockIdx.x == 0)
        for (int64_t i = (n4 << 2) + threadIdx.x; i < per_sample; i += blockDim.x) {
            const float v = (xb[i] - mean) * inv;
            yb[i] = rnd ? round_tf32_rna(v) : v;
        }
}

// ------------------------------------------------------------------------- norm_act
constexpr int kMaxGroups = 8;

// Thread mapping: a thread owns ONE channel quad c (gamma / beta / LayerScale loaded once) and walks over pixels
// (t, then output rows) with a fixed stride -- no per-element index arithmetic, 16-byte accesses, consecutive lanes on
// consecutive channel quads of the same pixel (then the next pixel), i.e. fully coalesced.
template <int OP, typename TO, typename TI>
__global__ void __launch_bounds__(256) norm_act_kernel(const TI* x, const double* __restrict__ stats,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       const float* __restrict__ snake_a, const float* __restrict__ scale,
                                                       const TO* residual, TO* y,
                                                       const aero_norm_act_params p) {
    constexpr bool GLU = (OP == AERO_NA_GLU || OP == AERO_NA_GLU_SCALE_RES);
    // grid = (chunks, segments): the chunks of one segment are scheduled together; AERO_TG_REVERSE walks both from the end
    const bool rev = p.flags & AERO_TG_REVERSE;
    const int seg = rev ? gridDim.y - 1 - blockIdx.y : blockIdx.y;      // scope 1: b ; scope 2: b*F_in + f
    const int chunk = rev ? gridDim.x - 1 - blockIdx.x : blockIdx.x;
    __shared__ float s_mean[kMaxGroups], s_rstd[kMaxGroups];
    if (threadIdx.x < p.groups) {
        const double n = (p.scope == 1) ? (double)p.F_in * p.T * (p.C / p.groups) : (double)p.T * p.C;
        const int64_t slot = (int64_t)seg * p.groups + threadIdx.x;
        const double mean = stats[2 * slot] / n;
        double var = stats[2 * slot + 1] / n - mean * mean;
        if (var < 0) var = 0;
        s_mean[threadIdx.x] = (float)mean;
        s_rstd[threadIdx.x] = (float)(1.0 / sqrt(var + (double)p.eps));
    }
    __syncthreads();
    const int Cout = GLU ? p.C / 2 : p.C;
    const int c4n = Cout >> 2;
    const int ppp = 256 / c4n;                        // pixels per pass of the CTA (host guarantees c4n <= 256)
    const int cq = threadIdx.x % c4n, dp = threadIdx.x / c4n;
    if (dp >= ppp) return;
    const int c = cq * 4;
    const int gw = p.C / p.groups;
    int b, f_lo, f_hi;                                // output rows handled by this segment
    if (p.scope == 1) { b = seg; f_lo = 0; f_hi = p.F_out; } else { b = seg / p.F_in; f_lo = seg % p.F_in; f_hi = f_lo + 1; }

    // per-channel constants: y = (x - m) * r * gamma + beta  ==  x * k + o
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c);
    const float4 be = *reinterpret_cast<const float4*>(beta + c);
    const float m0 = s_mean[c / gw], r0 = s_rstd[c / gw];
    const float4 k0 = make_float4(r0 * ga.x, r0 * ga.y, r0 * ga.z, r0 * ga.w);
    const float4 o0 = make_float4(be.x - m0 * k0.x, be.y - m0 * k0.y, be.z - m0 * k0.z, be.w - m0 * k0.w);
    float4 k1 = k0, o1 = o0, sc = make_float4(1.f, 1.f, 1.f, 1.f);
    if (GLU) {
        const int c2 = c + Cout;
        const float4 ga2 = *reinterpret_cast<const float4*>(gamma + c2);
        const float4 be2 = *reinterpret_cast<const float4*>(beta + c2);
        const float m1 = s_mean[c2 / gw], r1 = s_rstd[c2 / gw];
        k1 = make_float4(r1 * ga2.x, r1 * ga2.y, r1 * ga2.z, r1 * ga2.w);
        o1 = make_float4(be2.x - m1 * k1.x, be2.y - m1 * k1.y, be2.z - m1 * k1.z, be2.w - m1 * k1.w);
        if (OP == AERO_NA_GLU_SCALE_RES) sc = *reinterpret_cast<const float4*>(scale + c);
    }
    const bool rnd = (p.flags & AERO_TG_ROUND_TF32) && sizeof(TO) == 4;
    const int64_t npix = (int64_t)(f_hi - f_lo) * p.T;                       // pixels of this segment (row-major f, t)
    // one pixel: normalise, activate, store (loads are issued by the caller so that two pixels' worth are in flight)
    auto finish = [&](const float4 v, const float4 v2, const float4 rs, int fin, int64_t oidx) {
        float a[4] = {fmaf(v.x, k0.x, o0.x), fmaf(v.y, k0.y, o0.y), fmaf(v.z, k0.z, o0.z), fmaf(v.w, k0.w, o0.w)};
        float o[4];
        if (GLU) {
            const float gt[4] = {fmaf(v2.x, k1.x, o1.x), fmaf(v2.y, k1.y, o1.y), fmaf(v2.z, k1.z, o1.z), fmaf(v2.w, k1.w, o1.w)};
#pragma unroll
            for (int u = 0; u < 4; ++u) o[u] = a[u] * sigmoid_f(gt[u]);
            if (OP == AERO_NA_GLU_SCALE_RES) {
                o[0] = fmaf(sc.x, o[0], rs.x); o[1] = fmaf(sc.y, o[1], rs.y);
                o[2] = fmaf(sc.z, o[2], rs.z); o[3] = fmaf(sc.w, o[3], rs.w);
            }
        } else if (OP == AERO_NA_GELU) {
#pragma unroll
            for (int u = 0; u < 4; ++u) o[u] = gelu_exact(a[u]);
        } else if (OP == AERO_NA_RELU) {
#pragma unroll
            for (int u = 0; u < 4; ++u) o[u] = fmaxf(a[u], 0.f);
        } else if (OP == AERO_NA_SNAKE) {
            const float al = snake_a[fin];
            const float ia = 1.0f / al;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float sn = sinf(a[u] * al);
                o[u] = a[u] + ia * sn * sn;
            }
        } else {
#pragma unroll
            for (int u = 0; u < 4; ++u) o[u] = a[u];
        }
        if (rnd) {
#pragma unroll
            for (int u = 0; u < 4; ++u) o[u] = round_tf32_rna(o[u]);
        }
        st4(y + oidx, make_float4(o[0], o[1], o[2], o[3]));
    };
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    const int64_t step = (int64_t)gridDim.x * ppp;
    PixelWalk pw;                                                            // (row, t) of the pixel; no per-pixel division
    pw.init((int64_t)chunk * ppp + dp, step, p.T, 1 << 30);
    int64_t pix = (int64_t)chunk * ppp + dp;
    for (; pix + step < npix; pix += 2 * step) {                             // two pixels per iteration
        const int fl0 = f_lo + pw.f, t0 = pw.t;
        pw.next();
        const int fl1 = f_lo + pw.f, t1 = pw.t;
        pw.next();
        const TI* xp0 = x + (((int64_t)b * p.F_in + fl0 + p.f_off) * p.T + t0) * p.C + c;
        const TI* xp1 = x + (((int64_t)b * p.F_in + fl1 + p.f_off) * p.T + t1) * p.C + c;
        const int64_t oi0 = (((int64_t)b * p.F_out + fl0) * p.T + t0) * Cout + c;
        const int64_t oi1 = (((int64_t)b * p.F_out + fl1) * p.T + t1) * Cout + c;
        const float4 va = ld4(xp0), vb = ld4(xp1);
        const float4 va2 = GLU ? ld4(xp0 + Cout) : zero4;
        const float4 vb2 = GLU ? ld4(xp1 + Cout) : zero4;
        const float4 ra = (OP == AERO_NA_GLU_SCALE_RES) ? ld4(residual + oi0) : zero4;
        const float4 rb = (OP == AERO_NA_GLU_SCALE_RES) ? ld4(residual + oi1) : zero4;
        finish(va, va2, ra, fl0 + p.f_off, oi0);
        finish(vb, vb2, rb, fl1 + p.f_off, oi1);
    }
    if (pix < npix) {
        const int fl0 = f_lo + pw.f, t0 = pw.t;
        const TI* xp0 = x + (((int64_t)b * p.F_in + fl0 + p.f_off) * p.T + t0) * p.C + c;
        const int64_t oi0 = (((int64_t)b * p.F_out + fl0) * p.T + t0) * Cout + c;
        const float4 va = ld4(xp0);
        const float4 va2 = GLU ? ld4(xp0 + Cout) : zero4;
        const float4 ra = (OP == AERO_NA_GLU_SCALE_RES) ? ld4(residual + oi0) : zero4;
        finish(va, va2, ra, fl0 + p.f_off, oi0);
    }
}

}  // namespace aero

extern "C" int aero_sample_norm_fwd(const float* x, const double* stats, float* y, float* samp_affine, int32_t B,
                                    int64_t count, int64_t extent, int32_t round_tf32, aero_stream_t stream) {
    using namespace aero;
    const int64_t per_sample = extent > 0 ? extent : count;
    AERO_REQUIRE(x && stats && y && B >= 1 && count >= 2 && per_sample >= count, "aero_sample_norm_fwd: bad argument");
    AERO_REQUIRE((per_sample & 3) == 0 && (((uintptr_t)x | (uintptr_t)y) & 15) == 0,
                 "aero_sample_norm_fwd: per_sample must be a multiple of 4 and buffers 16-byte aligned");
    const int chunks = (int)((per_sample / 4 + 256 * 8 - 1) / (256 * 8));
    dim3 grid(chunks < 1 ? 1 : chunks, B);
    sample_norm_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, stats, y, samp_affine, count, per_sample, round_tf32);
    return check_launch("aero_sample_norm_fwd");
}

extern "C" int aero_norm_act_fwd(const void* x, const double* stats, const float* gamma, const float* beta,
                                 const float* snake_a, const float* scale, const void* residual, void* y,
                                 const aero_norm_act_params* p, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && stats && gamma && beta && y && p, "aero_norm_act_fwd: null argument");
    AERO_REQUIRE(p->scope == 1 || p->scope == 2, "aero_norm_act_fwd: scope=%d", p->scope);
    AERO_REQUIRE(p->groups >= 1 && p->groups <= kMaxGroups && p->C % p->groups == 0 && (p->C / p->groups) % 4 == 0,
                 "aero_norm_act_fwd: C=%d groups=%d (group width must be a multiple of 4)", p->C, p->groups);
    AERO_REQUIRE(p->scope == 1 || (p->groups == 1 && p->f_off == 0 && p->F_in == p->F_out),
                 "aero_norm_act_fwd: per-row scope needs groups=1 and no crop");
    AERO_REQUIRE(p->f_off >= 0 && p->f_off + p->F_out <= p->F_in, "aero_norm_act_fwd: crop out of range");
    const bool glu = (p->op == AERO_NA_GLU || p->op == AERO_NA_GLU_SCALE_RES);
    AERO_REQUIRE(!glu || p->C % 8 == 0, "aero_norm_act_fwd: GLU needs C %% 8 == 0");
    AERO_REQUIRE(p->op != AERO_NA_SNAKE || snake_a, "aero_norm_act_fwd: snake needs a[]");
    AERO_REQUIRE(p->op != AERO_NA_GLU_SCALE_RES || (scale && residual), "aero_norm_act_fwd: missing scale/residual");
    const int Cout = glu ? p->C / 2 : p->C;
    AERO_REQUIRE(Cout / 4 <= 256, "aero_norm_act_fwd: at most 1024 output channels (got %d)", Cout);
    const int ppp = 256 / (Cout / 4);
    const int64_t npix = (p->scope == 1 ? (int64_t)p->F_out * p->T : (int64_t)p->T);
    const int nseg = p->scope == 1 ? p->B : p->B * p->F_in;
    // ~8 pixels per thread; keep at least a few CTAs per SM in flight across all segments
    int chunks = (int)((npix + (int64_t)ppp * 8 - 1) / ((int64_t)ppp * 8));
    if (chunks < 1) chunks = 1;
    AERO_REQUIRE(nseg <= 65535, "aero_norm_act_fwd: at most 65535 segments (got %d)", nseg);
    dim3 grid(chunks, nseg);
    cudaStream_t st = (cudaStream_t)stream;
    const bool o16 = p->flags & AERO_TG_OUT_F16, i16 = p->flags & AERO_TG_A_F16;
    AERO_REQUIRE(!i16 || o16, "aero_norm_act_fwd: an FP16 input goes with an FP16 output");
#define AERO_NA_LAUNCH(OP)                                                                                                  \
    if (i16) norm_act_kernel<OP, __half, __half><<<grid, 256, 0, st>>>((const __half*)x, stats, gamma, beta, snake_a, scale, (const __half*)residual, (__half*)y, *p); \
    else if (o16) norm_act_kernel<OP, __half, float><<<grid, 256, 0, st>>>((const float*)x, stats, gamma, beta, snake_a, scale, (const __half*)residual, (__half*)y, *p); \
    else norm_act_kernel<OP, float, float><<<grid, 256, 0, st>>>((const float*)x, stats, gamma, beta, snake_a, scale, (const float*)residual, (float*)y, *p)
    switch (p->op) {
        case AERO_NA_NONE: AERO_NA_LAUNCH(AERO_NA_NONE); break;
        case AERO_NA_GELU: AERO_NA_LAUNCH(AERO_NA_GELU); break;
        case AERO_NA_GLU: AERO_NA_LAUNCH(AERO_NA_GLU); break;
        case AERO_NA_SNAKE: AERO_NA_LAUNCH(AERO_NA_SNAKE); break;
        case AERO_NA_RELU: AERO_NA_LAUNCH(AERO_NA_RELU); break;
        case AERO_NA_GLU_SCALE_RES: AERO_NA_LAUNCH(AERO_NA_GLU_SCALE_RES); break;
        default: set_error("aero_norm_act_fwd: op=%d", p->op); return AERO_ERR_INVALID;
    }
#undef AERO_NA_LAUNCH
    return check_launch("aero_norm_act_fwd");
}
