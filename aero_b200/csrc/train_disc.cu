// MelGAN multi-scale discriminator kernels (SURVEY.md section 8f rank 3; reference src/models/discriminators.py:14-78,
// src/models/modules.py WNConv1d): the grouped, strided 1-D convolutions (k = 41, stride 4, groups = C_in / 4) that cuDNN serves
// poorly -- forward, data gradient and weight gradient -- and weight normalisation (w = g * v / ||v||) forward / backward.
// Activations are channels-last [B][T][C] like everywhere else in the library; the dense layers of the discriminator (k = 15, 5, 3)
// run on the tap-GEMM.  fp32.
#include "common.cuh"

namespace aero {

constexpr int kGcCo = 64;       // output channels per CTA
constexpr int kGcT = 32;        // output time steps per CTA (forward / wgrad)

struct GconvP {
    int B, Tin, Tout, Cin, Cout, groups, k, stride, pad;
};

// y[b][to][co] = bias[co] + sum_{c < cpg, j < k} x[b][to*stride + j - pad][g*cpg + c] * w[co][c][j],  g = co / (Cout/groups)
__global__ void __launch_bounds__(256) gconv_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                        float* __restrict__ y, const GconvP p) {
    extern __shared__ float sm[];
    const int cpg = p.Cin / p.groups, opg = p.Cout / p.groups;
    const int co0 = blockIdx.x * kGcCo, to0 = blockIdx.y * kGcT, b = blockIdx.z;
    const int nco = min(kGcCo, p.Cout - co0);
    const int g0 = co0 / opg, ng = (co0 + nco - 1) / opg - g0 + 1;      // groups touched by this tile
    const int nch = ng * cpg;                                           // input channels needed
    const int win = (kGcT - 1) * p.stride + p.k;                        // input time steps needed
    float* ws = sm;                                                     // [nco][cpg*k]
    float* xs = sm + kGcCo * cpg * p.k;                                 // [win][nch]
    const int wl = cpg * p.k;
    for (int i = threadIdx.x; i < nco * wl; i += 256) ws[i] = w[(int64_t)co0 * wl + i];
    const int ti0 = to0 * p.stride - p.pad;
    for (int i = threadIdx.x; i < win * nch; i += 256) {
        const int tt = i / nch, c = i - tt * nch;
        const int ti = ti0 + tt;
        xs[i] = (ti >= 0 && ti < p.Tin) ? x[((int64_t)b * p.Tin + ti) * p.Cin + g0 * cpg + c] : 0.f;
    }
    __syncthreads();
    for (int o = threadIdx.x; o < kGcT * nco; o += 256) {
        const int tl = o / nco, cl = o - tl * nco;
        const int to = to0 + tl;
        if (to >= p.Tout) continue;
        const int co = co0 + cl;
        const int gl = co / opg - g0;
        const float* wr = ws + cl * wl;
        const float* xr = xs + (tl * p.stride) * nch + gl * cpg;
        float acc = bias ? bias[co] : 0.f;
        for (int c = 0; c < cpg; ++c)
            for (int j = 0; j < p.k; ++j) acc = fmaf(xr[j * nch + c], wr[c * p.k + j], acc);
        y[((int64_t)b * p.Tout + to) * p.Cout + co] = acc;
    }
}

// dx[b][ti][ci] = sum_{co in group(ci)} sum_{j : (ti + pad - j) % stride == 0} dy[b][(ti + pad - j)/stride][co] * w[co][ci % cpg][j]
constexpr int kGdT = 128;       // input time steps per CTA
__global__ void __launch_bounds__(256) gconv_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx,
                                                          const GconvP p) {
    extern __shared__ float sm[];
    const int cpg = p.Cin / p.groups, opg = p.Cout / p.groups;
    const int gt = max(1, kGcCo / opg);                                 // groups per CTA
    const int g0 = blockIdx.x * gt, ti0 = blockIdx.y * kGdT, b = blockIdx.z;
    const int ng = min(gt, p.groups - g0);
    const int nco = ng * opg, nci = ng * cpg;
    const int wl = cpg * p.k;
    float* ws = sm;                                                     // [nco][cpg*k]
    float* ds = sm + kGcCo * wl;                                        // [rows][nco]
    for (int i = threadIdx.x; i < nco * wl; i += 256) ws[i] = w[(int64_t)g0 * opg * wl + i];
    // output rows that can touch ti in [ti0, ti0 + kGdT): to in [ceil((ti0 + pad - k + 1)/s), floor((ti0 + kGdT - 1 + pad)/s)]
    int to_lo = ti0 + p.pad - (p.k - 1);
    to_lo = to_lo <= 0 ? 0 : (to_lo + p.stride - 1) / p.stride;
    const int to_hi = min(p.Tout - 1, (ti0 + kGdT - 1 + p.pad) / p.stride);
    const int rows = max(0, to_hi - to_lo + 1);
    for (int i = threadIdx.x; i < rows * nco; i += 256) {
        const int r = i / nco, c = i - r * nco;
        ds[i] = dy[((int64_t)b * p.Tout + to_lo + r) * p.Cout + g0 * opg + c];
    }
    __syncthreads();
    for (int o = threadIdx.x; o < kGdT * nci; o += 256) {
        const int tl = o / nci, cl = o - tl * nci;
        const int ti = ti0 + tl;
        if (ti >= p.Tin) continue;
        const int gl = cl / cpg, c = cl - gl * cpg;
        float acc = 0.f;
        const int jr = (ti + p.pad) % p.stride;                         // j = jr, jr + s, ...
        for (int j = jr; j < p.k; j += p.stride) {
            const int to = (ti + p.pad - j) / p.stride;
            if (ti + p.pad - j < 0) break;
            if (to > to_hi || to < to_lo) continue;
            const float* dr = ds + (to - to_lo) * nco + gl * opg;
            const float* wr = ws + (gl * opg) * wl + c * p.k + j;
            for (int q = 0; q < opg; ++q) acc = fmaf(dr[q], wr[q * wl], acc);
        }
        dx[((int64_t)b * p.Tin + ti) * p.Cin + g0 * cpg + cl] = acc;
    }
}

// dw[co][c][j] += sum_{b, to} dy[b][to][co] * x[b][to*stride + j - pad][g*cpg + c]   (fp32 atomics over (b, time chunks))
__global__ void __launch_bounds__(256) gconv_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw,
                                                          const GconvP p, const int chunks) {
    extern __shared__ float sm[];
    const int cpg = p.Cin / p.groups, opg = p.Cout / p.groups;
    const int co0 = blockIdx.x * kGcCo;
    const int nco = min(kGcCo, p.Cout - co0);
    const int g0 = co0 / opg, ng = (co0 + nco - 1) / opg - g0 + 1;
    const int nch = ng * cpg;
    const int win = (kGcT - 1) * p.stride + p.k;
    float* dsm = sm;                                                    // [kGcT][nco]
    float* xs = sm + kGcT * kGcCo;                                      // [win][nch]
    // thread -> (co, c) pairs; each accumulates the k taps of its pairs
    const int npair = nco * cpg;
    float acc[2][41];
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int j = 0; j < 41; ++j) acc[u][j] = 0.f;
    const int tiles_t = (p.Tout + kGcT - 1) / kGcT;
    const int64_t n_tiles = (int64_t)p.B * tiles_t;
    for (int64_t tile = blockIdx.y; tile < n_tiles; tile += chunks) {
        const int b = (int)(tile / tiles_t), to0 = (int)(tile % tiles_t) * kGcT;
        __syncthreads();
        for (int i = threadIdx.x; i < kGcT * nco; i += 256) {
            const int tl = i / nco, cl = i - tl * nco;
            dsm[i] = (to0 + tl < p.Tout) ? dy[((int64_t)b * p.Tout + to0 + tl) * p.Cout + co0 + cl] : 0.f;
        }
        const int ti0 = to0 * p.stride - p.pad;
        for (int i = threadIdx.x; i < win * nch; i += 256) {
            const int tt = i / nch, c = i - tt * nch;
            const int ti = ti0 + tt;
            xs[i] = (ti >= 0 && ti < p.Tin) ? x[((int64_t)b * p.Tin + ti) * p.Cin + g0 * cpg + c] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int pr = threadIdx.x + u * 256;
            if (pr >= npair) continue;
            const int cl = pr / cpg, c = pr - cl * cpg;
            const int gl = (co0 + cl) / opg - g0;
            const float* xc = xs + gl * cpg + c;
            for (int tl = 0; tl < kGcT; ++tl) {
                const float d = dsm[tl * nco + cl];
                const float* xr = xc + (tl * p.stride) * nch;
#pragma unroll
                for (int j = 0; j < 41; ++j)
                    if (j < p.k) acc[u][j] = fmaf(d, xr[j * nch], acc[u][j]);
            }
        }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const int pr = threadIdx.x + u * 256;
        if (pr >= npair) continue;
        const int cl = pr / cpg, c = pr - cl * cpg;
        float* out = dw + ((int64_t)(co0 + cl) * cpg + c) * p.k;
#pragma unroll
        for (int j = 0; j < 41; ++j)
            if (j < p.k && acc[u][j] != 0.f) atomicAdd(out + j, acc[u][j]);
    }
}

// ------------------------------------------------------------------------------------------------------------------------------
// MelGAN's own shape -- k = 41, stride 4, pad 20, 4 input channels per group, 4 or 16 outputs per group -- register-tiled: the generic
// kernels above spend two shared-memory loads per FMA; these keep the input window (forward) / the gradient window (dgrad) of four
// consecutive steps in registers and read the weights as one float4 per 16 FMAs.
constexpr int kG4K = 41, kG4S = 4, kG4Pad = 20, kG4Cpg = 4;
constexpr int kG4Co = 64;                      // output channels per CTA
constexpr int kG4T = 64;                       // forward: output steps per CTA
constexpr int kG4Wl = kG4Cpg * kG4K;           // 164 weights per output channel
constexpr int kG4Ws = 68;                      // forward weight tile [164][68]: rows 16-byte aligned, stores 4-way conflicted at worst
constexpr int kG4Xw = 300;                     // forward input rows [channel][300 steps]: 4 rows apart = 16 banks apart

// forward: thread = 4 consecutive output channels (one group) x 4 consecutive output steps
__global__ void __launch_bounds__(256) gconv41_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                          float* __restrict__ y, const GconvP p) {
    extern __shared__ __align__(16) float sm[];
    const int opg = p.Cout / p.groups;
    const int co0 = blockIdx.x * kG4Co, to0 = blockIdx.y * kG4T, b = blockIdx.z;
    const int g0 = co0 / opg;
    const int nch = (kG4Co / opg) * kG4Cpg;                           // input channels of this tile (16 or 64)
    float* ws = sm;                                                   // [164][68]
    float* xs = sm + kG4Wl * kG4Ws;                                   // [nch][300]
    for (int i = threadIdx.x; i < kG4Co * kG4Wl; i += 256) {
        const int cl = i / kG4Wl, e = i - cl * kG4Wl;
        ws[e * kG4Ws + cl] = w[(int64_t)co0 * kG4Wl + i];
    }
    constexpr int win = (kG4T - 1) * kG4S + kG4K;                     // 293
    const int ti0 = to0 * kG4S - kG4Pad;
    for (int i = threadIdx.x; i < kG4Xw * nch; i += 256) {
        const int tt = i / nch, c = i - tt * nch;
        const int ti = ti0 + tt;
        xs[c * kG4Xw + tt] = (tt < win && ti >= 0 && ti < p.Tin) ? x[((int64_t)b * p.Tin + ti) * p.Cin + g0 * kG4Cpg + c] : 0.f;
    }
    __syncthreads();
    const int cq = threadIdx.x & 15, tq = threadIdx.x >> 4;
    const int cl = 4 * cq, tl0 = 4 * tq;
    const int gl = cl / opg;
    float acc[4][4];
    {
        const float4 bv = bias ? *reinterpret_cast<const float4*>(bias + co0 + cl) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < 4; ++u) { acc[u][0] = bv.x; acc[u][1] = bv.y; acc[u][2] = bv.z; acc[u][3] = bv.w; }
    }
#pragma unroll 1
    for (int c = 0; c < kG4Cpg; ++c) {
        float xw[56];                                                 // steps 16 tq .. 16 tq + 55 of input channel (gl, c)
        const float* xr = xs + (gl * kG4Cpg + c) * kG4Xw + kG4S * tl0;
#pragma unroll
        for (int i = 0; i < 14; ++i) {
            const float4 v = *reinterpret_cast<const float4*>(xr + 4 * i);
            xw[4 * i] = v.x; xw[4 * i + 1] = v.y; xw[4 * i + 2] = v.z; xw[4 * i + 3] = v.w;
        }
        const float* wr = ws + (c * kG4K) * kG4Ws + cl;
#pragma unroll
        for (int j = 0; j < kG4K; ++j) {
            const float4 wv = *reinterpret_cast<const float4*>(wr + j * kG4Ws);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float xv = xw[kG4S * u + j];
                acc[u][0] = fmaf(xv, wv.x, acc[u][0]);
                acc[u][1] = fmaf(xv, wv.y, acc[u][1]);
                acc[u][2] = fmaf(xv, wv.z, acc[u][2]);
                acc[u][3] = fmaf(xv, wv.w, acc[u][3]);
            }
        }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int to = to0 + tl0 + u;
        if (to < p.Tout)
            *reinterpret_cast<float4*>(y + ((int64_t)b * p.Tout + to) * p.Cout + co0 + cl) = make_float4(acc[u][0], acc[u][1], acc[u][2], acc[u][3]);
    }
}

// data gradient.  With ti = 4 m + r:  dx[4m + r][c] = sum_{q < opg} sum_{i} dy[m + 5 - i][q] * w[q][c][r + 4 i]   (i = 0 .. 10, j = r + 4i <= 40)
// thread = (group, residue r, 4 consecutive m) x the group's 4 input channels; the 14-step gradient window of one output channel sits in
// registers, the weights are read as float4 over c.
constexpr int kG4Dw = 164;                     // per-output-channel weights, re-laid as [j][c]
// pad that makes a per-group stride = 16 (mod 32) floats: two neighbouring groups then occupy opposite halves of the 32 banks
__host__ __device__ inline int g4_skew(int base) { return (48 - base % 32) % 32; }
__global__ void __launch_bounds__(256) gconv41_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx,
                                                            const GconvP p, const int m_cta, const int ds_w) {
    extern __shared__ __align__(16) float sm[];
    const int opg = p.Cout / p.groups;
    const int ngl = kG4Co / opg;                                      // groups per CTA (4 or 16)
    const int co0 = blockIdx.x * kG4Co, m0c = blockIdx.y * m_cta, b = blockIdx.z;
    const int g0 = co0 / opg;
    const int gstride_w = opg * kG4Dw + g4_skew(opg * kG4Dw);
    float* ws = sm;                                                   // [ngl][opg][41][4] (+ skew)
    float* ds = sm + ngl * gstride_w;                                 // [64 output channels][ds_w steps] (+ skew per group)
    const int gstride_d = opg * ds_w + g4_skew(opg * ds_w);
    for (int i = threadIdx.x; i < kG4Co * kG4Wl; i += 256) {
        const int cl = i / kG4Wl, e = i - cl * kG4Wl;                 // e = c * 41 + j
        const int c = e / kG4K, j = e - c * kG4K;
        const int gl = cl / opg, q = cl - gl * opg;
        ws[gl * gstride_w + q * kG4Dw + j * 4 + c] = w[(int64_t)co0 * kG4Wl + i];
    }
    // gradient steps m0c - 5 .. m0c + m_cta + 8 (ds index 0 = step m0c - 5)
    const int to_base = m0c - 5;
    for (int i = threadIdx.x; i < ds_w * kG4Co; i += 256) {
        const int tt = i / kG4Co, cl = i - tt * kG4Co;
        const int to = to_base + tt;
        const int gl = cl / opg, q = cl - gl * opg;
        ds[gl * gstride_d + q * ds_w + tt] = (to >= 0 && to < p.Tout) ? dy[((int64_t)b * p.Tout + to) * p.Cout + co0 + cl] : 0.f;
    }
    __syncthreads();
    const int r = threadIdx.x & 3, gl = (threadIdx.x >> 2) % ngl, mb = threadIdx.x / (4 * ngl);
    const int ml = 4 * mb;                                            // first m of this thread, relative to m0c
    float acc[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[u][c] = 0.f;
    const int ntap = (r == 0) ? 11 : 10;
#pragma unroll 1
    for (int q = 0; q < opg; ++q) {
        float dw_[16];                                                // steps (m0 - 5) .. (m0 + 10) of output channel (gl, q)
        const float* dr = ds + gl * gstride_d + q * ds_w + ml;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float4 v = *reinterpret_cast<const float4*>(dr + 4 * i);
            dw_[4 * i] = v.x; dw_[4 * i + 1] = v.y; dw_[4 * i + 2] = v.z; dw_[4 * i + 3] = v.w;
        }
        const float* wr = ws + gl * gstride_w + q * kG4Dw + r * 4;
#pragma unroll
        for (int i = 0; i < 11; ++i) {
            if (i < ntap) {
                const float4 wv = *reinterpret_cast<const float4*>(wr + 16 * i);        // j = r + 4 i
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float dv = dw_[u + 10 - i];                 // step m0 + u + 5 - i
                    acc[u][0] = fmaf(dv, wv.x, acc[u][0]);
                    acc[u][1] = fmaf(dv, wv.y, acc[u][1]);
                    acc[u][2] = fmaf(dv, wv.z, acc[u][2]);
                    acc[u][3] = fmaf(dv, wv.w, acc[u][3]);
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int ti = kG4S * (m0c + ml + u) + r;
        if (ti < p.Tin)
            *reinterpret_cast<float4*>(dx + ((int64_t)b * p.Tin + ti) * p.Cin + (g0 + gl) * kG4Cpg) = make_float4(acc[u][0], acc[u][1], acc[u][2], acc[u][3]);
    }
}

// weight gradient: thread = one (output channel, input channel of its group) pair, all 41 taps in registers; per 4 output steps it
// loads one float4 of the gradient and a 56-step input window (14 float4s) for 656 FMAs.  Split over (batch, time tiles) with fp32 atomics.
constexpr int kG4Dy = 68;                      // gradient tile rows [64 channels][68 steps]
__global__ void __launch_bounds__(256) gconv41_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw,
                                                            const GconvP p, const int chunks) {
    extern __shared__ __align__(16) float sm[];
    const int opg = p.Cout / p.groups;
    const int co0 = blockIdx.x * kG4Co;
    const int g0 = co0 / opg;
    const int nch = (kG4Co / opg) * kG4Cpg;
    float* dys = sm;                                                  // [64][68]
    float* xs = sm + kG4Co * kG4Dy;                                   // [nch][300]
    const int cl = threadIdx.x >> 2, c = threadIdx.x & 3;
    const int gl = cl / opg;
    float acc[kG4K];
#pragma unroll
    for (int j = 0; j < kG4K; ++j) acc[j] = 0.f;
    constexpr int win = (kG4T - 1) * kG4S + kG4K;
    const int tiles_t = (p.Tout + kG4T - 1) / kG4T;
    const int n_tiles = p.B * tiles_t;
    for (int tile = blockIdx.y; tile < n_tiles; tile += chunks) {
        const int b = tile / tiles_t, to0 = (tile - b * tiles_t) * kG4T;
        __syncthreads();
        for (int i = threadIdx.x; i < kG4T * kG4Co; i += 256) {
            const int tl = i / kG4Co, q = i - tl * kG4Co;
            dys[q * kG4Dy + tl] = (to0 + tl < p.Tout) ? dy[((int64_t)b * p.Tout + to0 + tl) * p.Cout + co0 + q] : 0.f;
        }
        const int ti0 = to0 * kG4S - kG4Pad;
        for (int i = threadIdx.x; i < kG4Xw * nch; i += 256) {
            const int tt = i / nch, ch = i - tt * nch;
            const int ti = ti0 + tt;
            xs[ch * kG4Xw + tt] = (tt < win && ti >= 0 && ti < p.Tin) ? x[((int64_t)b * p.Tin + ti) * p.Cin + g0 * kG4Cpg + ch] : 0.f;
        }
        __syncthreads();
        const float* dr = dys + cl * kG4Dy;
        const float* xr = xs + (gl * kG4Cpg + c) * kG4Xw;
#pragma unroll 1
        for (int tq = 0; tq < kG4T / 4; ++tq) {
            const float4 d4 = *reinterpret_cast<const float4*>(dr + 4 * tq);
            const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
            float xw[56];
#pragma unroll
            for (int i = 0; i < 14; ++i) {
                const float4 v = *reinterpret_cast<const float4*>(xr + 16 * tq + 4 * i);
                xw[4 * i] = v.x; xw[4 * i + 1] = v.y; xw[4 * i + 2] = v.z; xw[4 * i + 3] = v.w;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int j = 0; j < kG4K; ++j) acc[j] = fmaf(dv[u], xw[kG4S * u + j], acc[j]);
        }
    }
    float* out = dw + ((int64_t)(co0 + cl) * kG4Cpg + c) * kG4K;
#pragma unroll
    for (int j = 0; j < kG4K; ++j)
        if (acc[j] != 0.f) atomicAdd(out + j, acc[j]);
}

static bool gconv41_ok(const GconvP& p) {
    if (p.k != kG4K || p.stride != kG4S || p.pad != kG4Pad || p.Cin != p.groups * kG4Cpg || p.Cout % kG4Co) return false;
    const int opg = p.Cout / p.groups;
    return opg == 4 || opg == 16;
}

// weight normalisation, one CTA per output channel (row):  w = g * v / ||v||
__global__ void __launch_bounds__(256) weight_norm_fwd_kernel(const float* __restrict__ v, const float* __restrict__ g, float* __restrict__ w,
                                                              float* __restrict__ norms, int len) {
    __shared__ double red[8];
    const int r = blockIdx.x;
    const float* vr = v + (int64_t)r * len;
    double s = 0.0;
    for (int i = threadIdx.x; i < len; i += 256) s += (double)vr[i] * vr[i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += red[k];
    const float nrm = (float)sqrt(t);
    if (threadIdx.x == 0 && norms) norms[r] = nrm;
    const float k = g[r] / nrm;
    for (int i = threadIdx.x; i < len; i += 256) w[(int64_t)r * len + i] = vr[i] * k;
}

// dg = sum(dw * v) / ||v||;   dv = g / ||v|| * (dw - v * sum(dw * v) / ||v||^2)     (both ADDED to the outputs)
__global__ void __launch_bounds__(256) weight_norm_bwd_kernel(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ dw,
                                                              float* __restrict__ dv, float* __restrict__ dg, int len) {
    __shared__ double red[2][8];
    const int r = blockIdx.x;
    const float* vr = v + (int64_t)r * len;
    const float* dr = dw + (int64_t)r * len;
    double s = 0.0, d = 0.0;
    for (int i = threadIdx.x; i < len; i += 256) { s += (double)vr[i] * vr[i]; d += (double)vr[i] * dr[i]; }
    s = warp_sum(s); d = warp_sum(d);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s; red[1][threadIdx.x >> 5] = d; }
    __syncthreads();
    double ts = 0.0, td = 0.0;
    for (int k = 0; k < 8; ++k) { ts += red[0][k]; td += red[1][k]; }
    const double nrm = sqrt(ts);
    if (threadIdx.x == 0) dg[r] += (float)(td / nrm);
    const float a = (float)(g[r] / nrm), bq = (float)(td / ts);
    for (int i = threadIdx.x; i < len; i += 256) dv[(int64_t)r * len + i] += a * (dr[i] - vr[i] * bq);
}

static int gconv_check(const GconvP& p) {
    AERO_REQUIRE(p.B >= 1 && p.Tin >= 1 && p.Tout >= 1 && p.groups >= 1 && p.Cin % p.groups == 0 && p.Cout % p.groups == 0, "aero_gconv1d: sizes");
    AERO_REQUIRE(p.k >= 1 && p.k <= 41 && p.stride >= 1 && p.pad >= 0, "aero_gconv1d: k=%d (<= 41) stride=%d", p.k, p.stride);
    AERO_REQUIRE(p.Tout == (p.Tin + 2 * p.pad - p.k) / p.stride + 1, "aero_gconv1d: Tout=%d inconsistent", p.Tout);
    const int cpg = p.Cin / p.groups, opg = p.Cout / p.groups;
    AERO_REQUIRE(cpg <= 8 && (kGcCo % opg == 0 || opg % kGcCo == 0), "aero_gconv1d: %d inputs / %d outputs per group unsupported", cpg, opg);
    AERO_REQUIRE(p.B <= 65535, "aero_gconv1d: batch too large");
    return AERO_OK;
}

static size_t gconv_smem(const GconvP& p, int rows_extra) {
    const int cpg = p.Cin / p.groups, opg = p.Cout / p.groups;
    const int ng = kGcCo / opg + 1;
    const int win = (kGcT - 1) * p.stride + p.k;
    return sizeof(float) * ((size_t)kGcCo * cpg * p.k + (size_t)(win > rows_extra ? win : rows_extra) * (size_t)(ng * cpg > kGcCo ? ng * cpg : kGcCo) + kGcT * kGcCo);
}

}  // namespace aero

extern "C" int aero_gconv1d_fwd(const float* x, const float* w, const float* bias, float* y, int32_t B, int32_t Tin, int32_t Tout, int32_t Cin,
                                int32_t Cout, int32_t groups, int32_t k, int32_t stride, int32_t pad, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && w && y, "aero_gconv1d_fwd: null argument");
    const GconvP p{B, Tin, Tout, Cin, Cout, groups, k, stride, pad};
    int rc = gconv_check(p);
    if (rc != AERO_OK) return rc;
    if (gconv41_ok(p)) {
        const int nch = (kG4Co / (Cout / groups)) * kG4Cpg;
        const size_t smem4 = sizeof(float) * ((size_t)kG4Wl * kG4Ws + (size_t)nch * kG4Xw);
        cudaFuncSetAttribute(gconv41_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem4);
        dim3 grid4(Cout / kG4Co, cdiv(Tout, kG4T), B);
        gconv41_fwd_kernel<<<grid4, 256, smem4, (cudaStream_t)stream>>>(x, w, bias, y, p);
        return check_launch("aero_gconv1d_fwd(k41)");
    }
    const size_t smem = gconv_smem(p, 0);
    cudaFuncSetAttribute(gconv_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid(cdiv(Cout, kGcCo), cdiv(Tout, kGcT), B);
    gconv_fwd_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(x, w, bias, y, p);
    return check_launch("aero_gconv1d_fwd");
}

extern "C" int aero_gconv1d_dgrad(const float* dy, const float* w, float* dx, int32_t B, int32_t Tin, int32_t Tout, int32_t Cin, int32_t Cout,
                                  int32_t groups, int32_t k, int32_t stride, int32_t pad, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(dy && w && dx, "aero_gconv1d_dgrad: null argument");
    const GconvP p{B, Tin, Tout, Cin, Cout, groups, k, stride, pad};
    int rc = gconv_check(p);
    if (rc != AERO_OK) return rc;
    const int opg = Cout / groups;
    if (gconv41_ok(p)) {
        const int ngl = kG4Co / opg;
        const int m_cta = 4 * (256 / (4 * ngl));                          // 64 (opg 16) or 16 (opg 4) values of m = ti / 4 per CTA
        const int ds_w = m_cta + 20;                                      // steps m0 - 5 .. m0 + m_cta + 14; 84 / 36: transposing stores 4-way conflicted
        const size_t smem4 = sizeof(float) * ((size_t)ngl * (opg * kG4Dw + g4_skew(opg * kG4Dw)) + (size_t)ngl * (opg * ds_w + g4_skew(opg * ds_w)));
        cudaFuncSetAttribute(gconv41_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem4);
        dim3 grid4(Cout / kG4Co, cdiv(cdiv(Tin, kG4S), m_cta), B);
        gconv41_dgrad_kernel<<<grid4, 256, smem4, (cudaStream_t)stream>>>(dy, w, dx, p, m_cta, ds_w);
        return check_launch("aero_gconv1d_dgrad(k41)");
    }
    const int gt = kGcCo / opg > 0 ? kGcCo / opg : 1;
    const int rows = (kGdT + k) / stride + 2;
    const size_t smem = gconv_smem(p, rows) + sizeof(float) * (size_t)rows * kGcCo;
    cudaFuncSetAttribute(gconv_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid(cdiv(groups, gt), cdiv(Tin, kGdT), B);
    gconv_dgrad_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(dy, w, dx, p);
    return check_launch("aero_gconv1d_dgrad");
}

extern "C" int aero_gconv1d_wgrad(const float* x, const float* dy, float* dw, int32_t B, int32_t Tin, int32_t Tout, int32_t Cin, int32_t Cout,
                                  int32_t groups, int32_t k, int32_t stride, int32_t pad, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && dy && dw, "aero_gconv1d_wgrad: null argument");
    const GconvP p{B, Tin, Tout, Cin, Cout, groups, k, stride, pad};
    int rc = gconv_check(p);
    if (rc != AERO_OK) return rc;
    if (gconv41_ok(p)) {
        const int nch = (kG4Co / (Cout / groups)) * kG4Cpg;
        const size_t smem4 = sizeof(float) * ((size_t)kG4Co * kG4Dy + (size_t)nch * kG4Xw);
        cudaFuncSetAttribute(gconv41_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem4);
        const int n_tiles4 = B * cdiv(Tout, kG4T);
        int chunks4 = (132 * 4) / (Cout / kG4Co) + 1;
        if (chunks4 > n_tiles4) chunks4 = n_tiles4;
        if (chunks4 > 65535) chunks4 = 65535;
        dim3 grid4(Cout / kG4Co, chunks4);
        gconv41_wgrad_kernel<<<grid4, 256, smem4, (cudaStream_t)stream>>>(x, dy, dw, p, chunks4);
        return check_launch("aero_gconv1d_wgrad(k41)");
    }
    const int cpg = Cin / groups;
    AERO_REQUIRE(kGcCo * cpg <= 512, "aero_gconv1d_wgrad: at most 8 input channels per group");
    const size_t smem = gconv_smem(p, 0);
    cudaFuncSetAttribute(gconv_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int64_t n_tiles = (int64_t)B * cdiv(Tout, kGcT);
    int chunks = (132 * 4) / cdiv(Cout, kGcCo) + 1;
    if (chunks > n_tiles) chunks = (int)n_tiles;
    if (chunks > 65535) chunks = 65535;
    dim3 grid(cdiv(Cout, kGcCo), chunks);
    gconv_wgrad_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(x, dy, dw, p, chunks);
    return check_launch("aero_gconv1d_wgrad");
}

extern "C" int aero_weight_norm_fwd(const float* v, const float* g, float* w, int32_t rows, int32_t len, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(v && g && w && rows >= 1 && len >= 1, "aero_weight_norm_fwd: bad argument");
    weight_norm_fwd_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>(v, g, w, nullptr, len);
    return check_launch("aero_weight_norm_fwd");
}

extern "C" int aero_weight_norm_bwd(const float* v, const float* g, const float* dw, float* dv, float* dg, int32_t rows, int32_t len,
                                    aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(v && g && dw && dv && dg && rows >= 1 && len >= 1, "aero_weight_norm_bwd: bad argument");
    weight_norm_bwd_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>(v, g, dw, dv, dg, len);
    return check_launch("aero_weight_norm_bwd");
}
