// Fused STFT / iSTFT kernels for sm_90a.
//
// aero_stft_fwd  : reflect pad + framing + window + real FFT (N/2-point complex FFT in shared
//                  memory + split post-pass) + n_fft^-1/2 + Nyquist drop + strided (channels-last
//                  or planar-complex) store + per-sample {sum, sumsq}.
//                  Replaces torch.stft as called at reference src/models/spec.py:12-20.
// aero_istft_fwd : strided load + C2R FFT + window + overlap-add + 1/sum(w^2) + centre trim.
//                  Replaces torch.istft as called at reference src/models/spec.py:30-37.
//
// Both are HBM-bound (SURVEY.md 8d: 33.9 MB / 36.9 MB per B=32 forward, FFT flops negligible).
// A CTA owns a run of consecutive frames of one signal so that, for every frequency bin, the
// frames it writes (reads) are contiguous in memory: >=128 B segments for the model's layouts.
#include "common.cuh"
#include "fft.cuh"

namespace aero {

constexpr int kThreads = 256;

template <int LOGN>
struct StftCfg {
    static constexpr int N = 1 << LOGN;
    static constexpr int M = N / 2;
    static constexpr int FB = (4096 / M) > 32 ? 32 : (4096 / M);       // frames per CTA (32 KB of work)
};

// ---------------------------------------------------------------------------------- forward
// VL (ragged batch, aero_stft_varlen_fwd): signal `sig` holds lengths[b] valid samples in a row of p.length; it is zero
// padded to a multiple of hop, reflected at that padded end, and its frames at or past its own frame count are written as
// zeros.  p.flags is 0 there.
template <int LOGN, bool VL>
__device__ __forceinline__ void stft_block(const float* __restrict__ x, const float* __restrict__ window,
                                           float* __restrict__ z, double* __restrict__ stats,
                                           const int32_t* __restrict__ lengths, const aero_stft_params p) {
    using C = StftCfg<LOGN>;
    constexpr int N = C::N, M = C::M, FB = C::FB, LOGM = LOGN - 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* work = reinterpret_cast<float2*>(smem_raw);                 // [FB][M]
    float2* stage = work + FB * M;                                      // [M+1][FB]
    float2* twN = stage + (M + 1) * FB;                                 // [M]  exp(-2 pi i j / N)
    float* wpad = reinterpret_cast<float*>(twN + M);                    // [N]
    float* seg = wpad + N;                                              // [(FB-1)*hop + N]

    const int sig = blockIdx.y;
    const int t0 = blockIdx.x * FB;
    const int L_in = VL ? min(lengths[sig / p.channels], p.length) : p.length;
    const int L = VL ? L_in + (p.hop - L_in % p.hop) % p.hop : L_in;   // VL: zero padded to a multiple of hop
    const int nfr = min(FB, (VL ? 1 + L / p.hop : p.frames) - t0);
    if constexpr (VL) {
        // frames past this signal's own end: zeros (t0 + fr < p.frames)
        float* zs = z + (int64_t)(sig / p.channels) * p.z_stride_b + (int64_t)(sig % p.channels) * p.z_stride_c;
        const int nz = min(FB, p.frames - t0) - max(nfr, 0);
        for (int i = threadIdx.x; i < p.bins_out * nz; i += kThreads) {
            const int k = i / nz, fr = max(nfr, 0) + i - k * nz;
            *reinterpret_cast<float2*>(zs + (int64_t)k * p.z_stride_k + (int64_t)(t0 + fr) * p.z_stride_t) = make_float2(0.f, 0.f);
        }
        if (nfr <= 0) return;
    }

    for (int j = threadIdx.x; j < M; j += kThreads) {
        float s, c;
        sincospif(2.0f * (float)j / (float)N, &s, &c);
        twN[j] = make_float2(c, -s);
    }
    const int wl = (N - p.win) / 2;
    for (int n = threadIdx.x; n < N; n += kThreads) {
        const int k = n - wl;
        wpad[n] = (k >= 0 && k < p.win) ? window[k] : 0.0f;
    }
    const int seg_len = (nfr - 1) * p.hop + N;
    const float* xs = x + (int64_t)sig * p.length;                      // rows of p.length samples
    const int q0 = t0 * p.hop - N / 2;
    const bool zero_pad = p.flags & AERO_STFT_ZERO_PAD;
    for (int i = threadIdx.x; i < seg_len; i += kThreads) {
        int src = q0 + i;
        const bool inside = src >= 0 && src < L;
        if (src < 0) src = -src;
        if (src >= L) src = 2 * (L - 1) - src;
        if constexpr (VL) seg[i] = (src >= 0 && src < L_in) ? xs[src] : 0.f;   // hop padding (and out-of-contract lengths) read as zeros
        else seg[i] = (zero_pad && !inside) ? 0.f : xs[src];
    }
    __syncthreads();

    // windowed frames, even/odd packed, bit-reversed placement
    for (int i = threadIdx.x; i < nfr * M; i += kThreads) {
        const int fr = i / M, n = i - fr * M;
        const float* s = seg + fr * p.hop + 2 * n;
        const int r = __brev((unsigned)n) >> (32 - LOGM);
        work[fr * M + r] = make_float2(s[0] * wpad[2 * n], s[1] * wpad[2 * n + 1]);
    }
    __syncthreads();
    fft_inplace<LOGM, kThreads>(work, twN, nfr);

    // split post-pass: X[k] = Xe[k] + w^k Xo[k], X[M-k] = conj(Xe[k] - w^k Xo[k])
    const float scale = rsqrtf((float)N);
    for (int i = threadIdx.x; i < nfr * (M / 2 + 1); i += kThreads) {
        const int fr = i / (M / 2 + 1), k = i - fr * (M / 2 + 1);
        const float2 a = work[fr * M + k];
        const float2 bq = work[fr * M + ((M - k) & (M - 1))];
        const float2 xe = make_float2(0.5f * (a.x + bq.x), 0.5f * (a.y - bq.y));
        const float2 d = make_float2(0.5f * (a.x - bq.x), 0.5f * (a.y + bq.y));   // (Z[k]-conj(Z[M-k]))/2
        const float2 xo = make_float2(d.y, -d.x);                                  // * (-i)
        const float2 t = cmul(twN[k], xo);
        stage[k * FB + fr] = make_float2(scale * (xe.x + t.x), scale * (xe.y + t.y));
        stage[(M - k) * FB + fr] = make_float2(scale * (xe.x - t.x), -scale * (xe.y - t.y));
    }
    __syncthreads();

    float* zs = z + (int64_t)(sig / p.channels) * p.z_stride_b + (int64_t)(sig % p.channels) * p.z_stride_c;
    float lsum = 0.f, lsq = 0.f;
    for (int i = threadIdx.x; i < p.bins_out * nfr; i += kThreads) {
        const int k = i / nfr, fr = i - k * nfr;
        float2 v = stage[k * FB + fr];
        if (!VL && (p.flags & AERO_STFT_ADJ_SCALE)) {   // adjoint of the C2R transform: interior bins count twice, DC / Nyquist are real
            if (k == 0 || k == M) v.y = 0.f;
            else { v.x *= 2.0f; v.y *= 2.0f; }
        }
        *reinterpret_cast<float2*>(zs + (int64_t)k * p.z_stride_k + (int64_t)(t0 + fr) * p.z_stride_t) = v;
        lsum += v.x + v.y;
        lsq += v.x * v.x + v.y * v.y;
    }
    if (stats != nullptr) {
        __shared__ double red[2][kThreads / 32];
        double ds = warp_sum((double)lsum), dq = warp_sum((double)lsq);
        if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = ds; red[1][threadIdx.x >> 5] = dq; }
        __syncthreads();
        if (threadIdx.x == 0) {
            double a = 0, b = 0;
            for (int w = 0; w < kThreads / 32; ++w) { a += red[0][w]; b += red[1][w]; }
            atomicAdd(&stats[2 * (sig / p.channels)], a);
            atomicAdd(&stats[2 * (sig / p.channels) + 1], b);
        }
    }
}

template <int LOGN>
__global__ void __launch_bounds__(kThreads) stft_kernel(const float* __restrict__ x, const float* __restrict__ window,
                                                        float* __restrict__ z, double* __restrict__ stats,
                                                        const aero_stft_params p) {
    stft_block<LOGN, false>(x, window, z, stats, nullptr, p);
}

template <int LOGN>
__global__ void __launch_bounds__(kThreads) stft_varlen_kernel(const float* __restrict__ x, const float* __restrict__ window,
                                                               float* __restrict__ z, double* __restrict__ stats,
                                                               const int32_t* __restrict__ lengths, const aero_stft_params p) {
    stft_block<LOGN, true>(x, window, z, stats, lengths, p);
}

// The entry point a launch serves, named in its errors: per-clip lengths (or frame counts) select the ragged one.
static const char* stft_entry(const void* per_clip) { return per_clip ? "aero_stft_varlen_fwd" : "aero_stft_fwd"; }
static const char* istft_entry(const void* per_clip) { return per_clip ? "aero_istft_varlen_fwd" : "aero_istft_fwd"; }

// lengths == nullptr: fixed-length stft_kernel, otherwise stft_varlen_kernel.
template <int LOGN>
static int launch_stft(const float* x, const float* window, float* z, double* stats, const int32_t* lengths,
                       const aero_stft_params& p, cudaStream_t st) {
    using C = StftCfg<LOGN>;
    const size_t smem = sizeof(float2) * (C::FB * C::M + (C::M + 1) * C::FB + C::M) +
                        sizeof(float) * (C::N + (size_t)(C::FB - 1) * p.hop + C::N);
    if (smem > 227 * 1024) {
        set_error("%s: hop %d too large for n_fft %d (smem %zu)", stft_entry(lengths), p.hop, p.n_fft, smem);
        return AERO_ERR_UNSUPPORTED;
    }
    dim3 grid(cdiv(p.frames, C::FB), p.n_signals);
    if (lengths) {
        cudaFuncSetAttribute(stft_varlen_kernel<LOGN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        stft_varlen_kernel<LOGN><<<grid, kThreads, smem, st>>>(x, window, z, stats, lengths, p);
    } else {
        cudaFuncSetAttribute(stft_kernel<LOGN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        stft_kernel<LOGN><<<grid, kThreads, smem, st>>>(x, window, z, stats, p);
    }
    return check_launch(stft_entry(lengths));
}

// ---------------------------------------------------------------------------------- inverse
template <int LOGN>
struct IstftCfg {
    static constexpr int N = 1 << LOGN;
    static constexpr int M = N / 2;
    static constexpr int NF = (8192 / M) > 32 ? 32 : ((8192 / M) < 12 ? 12 : (8192 / M));   // frames resident per CTA (64 KB; >= 12 so that
                                                                                             // n_fft 2048 / hop 240 of the MR-STFT loss fits)
};

// VL (ragged batch, aero_istft_varlen_fwd): signal `sig` uses its own frames[b] frames and writes out_lens[b] samples of
// its row of p.out_len; the rest of the row is zeroed.
template <int LOGN, bool VL>
__device__ __forceinline__ void istft_block(const float* __restrict__ z, const float* __restrict__ window,
                                            float* __restrict__ y, const aero_istft_params& p,
                                            const int OB, const int halo, const int32_t* __restrict__ frames_b,
                                            const int32_t* __restrict__ out_lens) {
    using C = IstftCfg<LOGN>;
    constexpr int N = C::N, M = C::M, NF = C::NF, LOGM = LOGN - 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* work = reinterpret_cast<float2*>(smem_raw);                 // [NF][M]  (later: [NF][N] real frames)
    float2* xs = work + NF * M;                                         // [NF][M+1] spectra
    float2* twN = xs + NF * (M + 1);                                    // [M] exp(+2 pi i j / N)
    float* wpad = reinterpret_cast<float*>(twN + M);                    // [N]

    const int sig = blockIdx.y;
    const int blk = blockIdx.x;
    int n_frames = p.frames, out_len = p.out_len;
    if constexpr (VL) {
        n_frames = frames_b[sig / p.channels];
        out_len = out_lens[sig / p.channels];
    }
    const int t_lo = max(0, blk * OB - halo);
    const int t_hi = min(n_frames - 1, blk * OB + OB - 1);
    const int nfr = t_hi - t_lo + 1;
    if constexpr (VL) {
        if (nfr <= 0) {              // entirely past this signal's end: its share of the row is padding
            float* ys = y + (int64_t)sig * p.out_len;
            for (int i = threadIdx.x; i < OB * p.hop; i += kThreads) {
                const int n_out = blk * OB * p.hop + i - N / 2;
                if (n_out >= out_len && n_out < p.out_len) ys[n_out] = 0.f;
            }
            return;
        }
    }

    for (int j = threadIdx.x; j < M; j += kThreads) {
        float s, c;
        sincospif(2.0f * (float)j / (float)N, &s, &c);
        twN[j] = make_float2(c, s);
    }
    const int wl = (N - p.win) / 2;
    for (int n = threadIdx.x; n < N; n += kThreads) {
        const int k = n - wl;
        wpad[n] = (k >= 0 && k < p.win) ? window[k] : 0.0f;
    }
    const float* zs = z + (int64_t)(sig / p.channels) * p.z_stride_b + (int64_t)(sig % p.channels) * p.z_stride_c;
    for (int i = threadIdx.x; i < (M + 1) * nfr; i += kThreads) {
        const int k = i / nfr, fr = i - k * nfr;
        float2 v = make_float2(0.f, 0.f);
        if (k < p.bins_in)
            v = *reinterpret_cast<const float2*>(zs + (int64_t)k * p.z_stride_k + (int64_t)(t_lo + fr) * p.z_stride_t);
        if (k == 0 || k == M) v.y = 0.f;       // C2R ignores the imaginary part of DC and Nyquist
        xs[fr * (M + 1) + k] = v;
    }
    __syncthreads();

    // Y[k] = Xe[k] + i Xo[k];  Xe = (X[k]+conj(X[M-k]))/2,  Xo = conj(w^k) (X[k]-conj(X[M-k]))/2
    for (int i = threadIdx.x; i < nfr * M; i += kThreads) {
        const int fr = i / M, k = i - fr * M;
        const float2 a = xs[fr * (M + 1) + k];
        const float2 b = xs[fr * (M + 1) + (M - k)];
        const float2 xe = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y - b.y));
        const float2 d = make_float2(0.5f * (a.x - b.x), 0.5f * (a.y + b.y));
        const float2 xo = cmul(twN[k], d);                              // twN holds exp(+i..) = conj(w^k)
        const int r = __brev((unsigned)k) >> (32 - LOGM);
        work[fr * M + r] = make_float2(xe.x - xo.y, xe.y + xo.x);      // xe + i*xo
    }
    __syncthreads();
    fft_inplace<LOGM, kThreads>(work, twN, nfr);

    // overlap-add; work now holds real frames: frame fr, sample n at ((float*)work)[fr*N + n]
    const float* frames = reinterpret_cast<const float*>(work);
    const float scale = 2.0f * rsqrtf((float)N);                        // sqrt(N) / M
    const int p0 = blk * OB * p.hop;
    const int span = OB * p.hop;
    float* ys = y + (int64_t)sig * p.out_len;
    const bool raw = p.flags & AERO_ISTFT_RAW;                          // no centre trim, no envelope division (adjoint of the STFT)
    for (int i = threadIdx.x; i < span; i += kThreads) {
        const int pos = p0 + i;
        const int n_out = raw ? pos : pos - N / 2;
        if (n_out < 0 || n_out >= p.out_len) continue;
        if constexpr (VL) {
            if (n_out >= out_len) { ys[n_out] = 0.f; continue; }
        }
        int ta = (pos - N + p.hop) / p.hop;                             // ceil((pos-N+1)/hop) for pos-N+1 > 0
        if (pos - N + 1 <= 0) ta = 0;
        ta = max(ta, t_lo);
        const int tb = min(pos / p.hop, t_hi);
        float acc = 0.f, env = 0.f;
        for (int t = ta; t <= tb; ++t) {
            const int n = pos - t * p.hop;
            const float w = wpad[n];
            acc += frames[(t - t_lo) * N + n] * w;
            env += w * w;
        }
        ys[n_out] = raw ? acc * scale : acc * scale / env;
    }
}

template <int LOGN>
__global__ void __launch_bounds__(kThreads) istft_kernel(const float* __restrict__ z, const float* __restrict__ window,
                                                         float* __restrict__ y, const aero_istft_params p,
                                                         const int OB, const int halo) {
    istft_block<LOGN, false>(z, window, y, p, OB, halo, nullptr, nullptr);
}

template <int LOGN>
__global__ void __launch_bounds__(kThreads) istft_varlen_kernel(const float* __restrict__ z, const float* __restrict__ window,
                                                                float* __restrict__ y, const aero_istft_params p,
                                                                const int OB, const int halo, const int32_t* __restrict__ frames,
                                                                const int32_t* __restrict__ out_lens) {
    istft_block<LOGN, true>(z, window, y, p, OB, halo, frames, out_lens);
}

// frames == nullptr: fixed-length istft_kernel, otherwise istft_varlen_kernel with per-signal frame counts and output lengths.
template <int LOGN>
static int launch_istft(const float* z, const float* window, float* y, const int32_t* frames, const int32_t* out_lens,
                        const aero_istft_params& p, cudaStream_t st) {
    using C = IstftCfg<LOGN>;
    const int halo = (C::N - 1) / p.hop;
    const int OB = C::NF - halo;
    if (OB < 1) {
        set_error("%s: hop %d too small for n_fft %d (needs hop >= n_fft/%d)", istft_entry(frames), p.hop, p.n_fft, C::NF - 1);
        return AERO_ERR_UNSUPPORTED;
    }
    const size_t smem = sizeof(float2) * (C::NF * C::M + C::NF * (C::M + 1) + C::M) + sizeof(float) * C::N;
    if (smem > 227 * 1024) {
        set_error("%s: n_fft %d needs %zu bytes of shared memory", istft_entry(frames), p.n_fft, smem);
        return AERO_ERR_UNSUPPORTED;
    }
    // padded positions that can produce output: [N/2, N/2 + out_len)  (raw mode: [0, out_len))
    const int last_pos = ((p.flags & AERO_ISTFT_RAW) ? 0 : C::N / 2) + p.out_len - 1;
    dim3 grid(last_pos / (OB * p.hop) + 1, p.n_signals);
    if (frames) {
        cudaFuncSetAttribute(istft_varlen_kernel<LOGN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        istft_varlen_kernel<LOGN><<<grid, kThreads, smem, st>>>(z, window, y, p, OB, halo, frames, out_lens);
    } else {
        cudaFuncSetAttribute(istft_kernel<LOGN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        istft_kernel<LOGN><<<grid, kThreads, smem, st>>>(z, window, y, p, OB, halo);
    }
    return check_launch(istft_entry(frames));
}

// ---------------------------------------------------------------------------------- n_fft = 512 fast path
// The model's size.  The 256-point complex FFT behind the 512-point real transform is done as a four-step 16 x 16
// decomposition with both 16-point FFTs held entirely in registers (two radix-4 passes, constant twiddles):
//   n = 16 n1 + n2, k = k1 + 16 k2:  Z[k] = sum_n2 W256^(n2 k1) [ sum_n1 z[16 n1 + n2] W16^(n1 k1) ] W16^(n2 k2)
// One thread owns one (frame, n2) column in pass 1 and one (frame, k1) row in pass 2; 16 frames per CTA = 256 threads;
// four block barriers in total (the radix-2 kernel above needs eleven), no bit reversal.
template <bool INV>
__device__ __forceinline__ void dft4(float2& a0, float2& a1, float2& a2, float2& a3) {
    const float2 s02 = make_float2(a0.x + a2.x, a0.y + a2.y), d02 = make_float2(a0.x - a2.x, a0.y - a2.y);
    const float2 s13 = make_float2(a1.x + a3.x, a1.y + a3.y), d13 = make_float2(a1.x - a3.x, a1.y - a3.y);
    // forward: y1 = d02 - i d13, y3 = d02 + i d13; inverse: swapped
    const float2 jd = INV ? make_float2(-d13.y, d13.x) : make_float2(d13.y, -d13.x);      // (-/+ i) * d13
    a0 = make_float2(s02.x + s13.x, s02.y + s13.y);
    a2 = make_float2(s02.x - s13.x, s02.y - s13.y);
    a1 = make_float2(d02.x + jd.x, d02.y + jd.y);
    a3 = make_float2(d02.x - jd.x, d02.y - jd.y);
}

// in-register 16-point DFT; on return v[r + 4 s] holds A[r + 4 s] (natural order)
template <bool INV>
__device__ __forceinline__ void dft16(float2 (&v)[16]) {
    // n = 4 p + q, k = r + 4 s.  Step 1: 4-point DFT over p for each q: (v[q], v[4+q], v[8+q], v[12+q]) -> B[q][r] stored at v[4 r + q]
#pragma unroll
    for (int q = 0; q < 4; ++q) dft4<INV>(v[q], v[4 + q], v[8 + q], v[12 + q]);
    // Step 2: twiddle B[q][r] *= W16^(q r)
    constexpr float C1 = 0.92387953251128674f, S1 = 0.38268343236508977f, C2 = 0.70710678118654752f;
    const float sg = INV ? 1.f : -1.f;                   // forward twiddles have negative imaginary part
    // (q, r) pairs with q r in {1,2,3,4,6,9}
    v[4 * 1 + 1] = cmul(v[4 * 1 + 1], make_float2(C1, sg * S1));      // q r = 1
    v[4 * 1 + 2] = cmul(v[4 * 1 + 2], make_float2(C2, sg * C2));      // 2  (r=1,q=2)
    v[4 * 2 + 1] = cmul(v[4 * 2 + 1], make_float2(C2, sg * C2));      // 2  (r=2,q=1)
    v[4 * 1 + 3] = cmul(v[4 * 1 + 3], make_float2(S1, sg * C1));      // 3  (r=1,q=3)
    v[4 * 3 + 1] = cmul(v[4 * 3 + 1], make_float2(S1, sg * C1));      // 3  (r=3,q=1)
    v[4 * 2 + 2] = cmul(v[4 * 2 + 2], make_float2(0.f, sg * 1.f));     // 4  (r=2,q=2)
    v[4 * 2 + 3] = cmul(v[4 * 2 + 3], make_float2(-C2, sg * C2));      // 6  (r=2,q=3)
    v[4 * 3 + 2] = cmul(v[4 * 3 + 2], make_float2(-C2, sg * C2));      // 6  (r=3,q=2)
    v[4 * 3 + 3] = cmul(v[4 * 3 + 3], make_float2(-C1, -sg * S1));     // 9  (r=3,q=3): cos(9pi/8) = -C1, sin = -S1
    // Step 3: 4-point DFT over q for each r: (v[4r], v[4r+1], v[4r+2], v[4r+3]) -> A[r + 4 s] at v[4 r + s]
#pragma unroll
    for (int r = 0; r < 4; ++r) dft4<INV>(v[4 * r], v[4 * r + 1], v[4 * r + 2], v[4 * r + 3]);
    // reorder v[4 r + s] -> v[r + 4 s]  (4x4 transpose, register renaming only)
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int sx = r + 1; sx < 4; ++sx) { const float2 t = v[4 * r + sx]; v[4 * r + sx] = v[4 * sx + r]; v[4 * sx + r] = t; }
}

constexpr int kF512 = 16;            // frames per CTA
constexpr int kTPad = 17;            // padded row of the transpose buffer (float2)

// VL: the per-signal length handling of stft_block.
template <bool VL>
__device__ __forceinline__ void stft512_block(const float* __restrict__ x, const float* __restrict__ window,
                                              float* __restrict__ z, double* __restrict__ stats,
                                              const int32_t* __restrict__ lengths, const aero_stft_params p) {
    constexpr int N = 512, M = 256, ZP = 257;                           // ZP: padded frame pitch of Z (bank-conflict-free columns)
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* tbuf = reinterpret_cast<float2*>(smem_raw);                 // [16][16][17] pass-1 output, then Z [16][257] (same memory)
    float2* tw256 = tbuf + kF512 * 16 * kTPad;                          // [256] exp(-2 pi i m / 256)
    float2* twp = tw256 + M;                                            // [129] exp(-2 pi i k / 512)
    float* wpad = reinterpret_cast<float*>(twp + 132);                  // [512]
    float* seg = wpad + N;                                              // [15*hop + 512]

    const int sig = blockIdx.y;
    const int t0 = blockIdx.x * kF512;
    const int L_in = VL ? min(lengths[sig / p.channels], p.length) : p.length;
    const int L = VL ? L_in + (p.hop - L_in % p.hop) % p.hop : L_in;   // VL: zero padded to a multiple of hop
    const int nfr = min(kF512, (VL ? 1 + L / p.hop : p.frames) - t0);
    const int tid = threadIdx.x;
    if constexpr (VL) {
        // frames past this signal's own end: zeros (t0 + fr < p.frames)
        float* zs = z + (int64_t)(sig / p.channels) * p.z_stride_b + (int64_t)(sig % p.channels) * p.z_stride_c;
        const int nz = min(kF512, p.frames - t0) - max(nfr, 0);
        for (int i = tid; i < p.bins_out * nz; i += 256) {
            const int k = i / nz, fr = max(nfr, 0) + i - k * nz;
            *reinterpret_cast<float2*>(zs + (int64_t)k * p.z_stride_k + (int64_t)(t0 + fr) * p.z_stride_t) = make_float2(0.f, 0.f);
        }
        if (nfr <= 0) return;
    }
    {
        float sn, cs;
        sincospif(2.0f * (float)tid / 256.0f, &sn, &cs);
        tw256[tid] = make_float2(cs, -sn);
        if (tid <= 128) { sincospif(2.0f * (float)tid / 512.0f, &sn, &cs); twp[tid] = make_float2(cs, -sn); }
    }
    const int wl = (N - p.win) / 2;
    for (int n = tid; n < N; n += 256) { const int k = n - wl; wpad[n] = (k >= 0 && k < p.win) ? window[k] : 0.0f; }
    const int seg_len = (nfr - 1) * p.hop + N;
    const float* xs = x + (int64_t)sig * p.length;                      // rows of p.length samples
    const int q0 = t0 * p.hop - N / 2;
    for (int i = tid; i < seg_len; i += 256) {
        int src = q0 + i;
        if (src < 0) src = -src;
        if (src >= L) src = 2 * (L - 1) - src;
        if constexpr (VL) seg[i] = (src >= 0 && src < L_in) ? xs[src] : 0.f;   // hop padding (and out-of-contract lengths) read as zeros
        else seg[i] = xs[src];
    }
    __syncthreads();

    const int fr = tid >> 4, c = tid & 15;            // pass 1: c = n2; pass 2: c = k1
    float2 v[16];
    if (fr < nfr) {
        // z[n] = x[2n] w[2n] + i x[2n+1] w[2n+1], n = 16 n1 + n2
        const float2* sf = reinterpret_cast<const float2*>(seg + fr * p.hop);      // hop even (checked by the dispatcher)
        const float2* wf = reinterpret_cast<const float2*>(wpad);
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const float2 xv = sf[16 * n1 + c], wv = wf[16 * n1 + c];
            v[n1] = make_float2(xv.x * wv.x, xv.y * wv.y);
        }
        dft16<false>(v);
#pragma unroll
        for (int k1 = 0; k1 < 16; ++k1) tbuf[(fr * 16 + c) * kTPad + k1] = cmul(v[k1], tw256[c * k1]);
    }
    __syncthreads();
    if (fr < nfr) {
#pragma unroll
        for (int n2 = 0; n2 < 16; ++n2) v[n2] = tbuf[(fr * 16 + n2) * kTPad + c];
        dft16<false>(v);
    }
    __syncthreads();                                  // every thread has its pass-2 inputs in registers: reuse the buffer for Z
    float2* Z = tbuf;
    if (fr < nfr) {
#pragma unroll
        for (int k2 = 0; k2 < 16; ++k2) Z[fr * ZP + c + 16 * k2] = v[k2];
    }
    __syncthreads();

    // split post-pass fused with the store: X[k] = Xe[k] + w^k Xo[k], X[M-k] = conj(Xe[k] - w^k Xo[k]).
    // Consecutive lanes take consecutive frames of one bin: each bin row is a contiguous run in memory.
    float* zs = z + (int64_t)(sig / p.channels) * p.z_stride_b + (int64_t)(sig % p.channels) * p.z_stride_c;
    const float scale = rsqrtf((float)N);
    float lsum = 0.f, lsq = 0.f;
    for (int i = tid; i < (M / 2 + 1) * kF512; i += 256) {
        const int k = i >> 4, f2 = i & 15;
        if (f2 >= nfr) continue;
        const float2 a = Z[f2 * ZP + k];
        const float2 bq = Z[f2 * ZP + ((M - k) & (M - 1))];
        const float2 xe = make_float2(0.5f * (a.x + bq.x), 0.5f * (a.y - bq.y));
        const float2 d = make_float2(0.5f * (a.x - bq.x), 0.5f * (a.y + bq.y));
        const float2 xo = make_float2(d.y, -d.x);
        const float2 t = cmul(twp[k], xo);
        const float2 lo = make_float2(scale * (xe.x + t.x), scale * (xe.y + t.y));
        const float2 hi = make_float2(scale * (xe.x - t.x), -scale * (xe.y - t.y));
        float* dst = zs + (int64_t)(t0 + f2) * p.z_stride_t;
        if (k < p.bins_out) {
            *reinterpret_cast<float2*>(dst + (int64_t)k * p.z_stride_k) = lo;
            lsum += lo.x + lo.y; lsq += lo.x * lo.x + lo.y * lo.y;
        }
        if (k != M - k && (M - k) < p.bins_out) {
            *reinterpret_cast<float2*>(dst + (int64_t)(M - k) * p.z_stride_k) = hi;
            lsum += hi.x + hi.y; lsq += hi.x * hi.x + hi.y * hi.y;
        }
    }
    if (stats != nullptr) {
        __shared__ double red[2][8];
        double ds = warp_sum((double)lsum), dq = warp_sum((double)lsq);
        if ((tid & 31) == 0) { red[0][tid >> 5] = ds; red[1][tid >> 5] = dq; }
        __syncthreads();
        if (tid == 0) {
            double a = 0, b = 0;
            for (int w = 0; w < 8; ++w) { a += red[0][w]; b += red[1][w]; }
            atomicAdd(&stats[2 * (sig / p.channels)], a);
            atomicAdd(&stats[2 * (sig / p.channels) + 1], b);
        }
    }
}

__global__ void __launch_bounds__(256) stft512_kernel(const float* __restrict__ x, const float* __restrict__ window,
                                                      float* __restrict__ z, double* __restrict__ stats,
                                                      const aero_stft_params p) {
    stft512_block<false>(x, window, z, stats, nullptr, p);
}

__global__ void __launch_bounds__(256) stft512_varlen_kernel(const float* __restrict__ x, const float* __restrict__ window,
                                                             float* __restrict__ z, double* __restrict__ stats,
                                                             const int32_t* __restrict__ lengths, const aero_stft_params p) {
    stft512_block<true>(x, window, z, stats, lengths, p);
}

static int launch_stft512(const float* x, const float* window, float* z, double* stats, const int32_t* lengths,
                          const aero_stft_params& p, cudaStream_t st) {
    const size_t smem = sizeof(float2) * ((size_t)kF512 * 16 * kTPad + 256 + 132) +
                        sizeof(float) * (512 + (size_t)(kF512 - 1) * p.hop + 512);
    dim3 grid(cdiv(p.frames, kF512), p.n_signals);
    if (lengths) {
        cudaFuncSetAttribute(stft512_varlen_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        stft512_varlen_kernel<<<grid, 256, smem, st>>>(x, window, z, stats, lengths, p);
        return check_launch("aero_stft_varlen_fwd(512)");
    }
    cudaFuncSetAttribute(stft512_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    stft512_kernel<<<grid, 256, smem, st>>>(x, window, z, stats, p);
    return check_launch("aero_stft_fwd(512)");
}

// inverse: NF resident frames per CTA, same four-step transform with conjugate twiddles, then overlap-add.
// VL: per-signal frame counts and output lengths, as in istft_block.
constexpr int kI512 = 32;            // resident frames per CTA: 25 output hops per 32 transformed frames at hop = n_fft/8

template <int NF, bool VL>    // NF: resident frames per CTA (16 threads each)
__device__ __forceinline__ void istft512_block(const float* __restrict__ z, const float* __restrict__ window,
                                               float* __restrict__ y, const aero_istft_params p, const int OB,
                                               const int halo, const int32_t* __restrict__ frames_b,
                                               const int32_t* __restrict__ out_lens) {
    constexpr int N = 512, M = 256, NTH = NF * 16;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* xsb = reinterpret_cast<float2*>(smem_raw);                  // [16][257] spectra -> transpose buffer -> real frames [16][512]
    float2* tw256 = xsb + NF * 16 * kTPad;                              // [256] exp(+2 pi i m / 256)  (xsb region sized for the transpose)
    float2* twp = tw256 + M;                                            // [257] exp(+2 pi i k / 512), k <= 256
    float* wpad = reinterpret_cast<float*>(twp + 260);                  // [512]

    const int sig = blockIdx.y, blk = blockIdx.x, tid = threadIdx.x;
    const int n_frames = VL ? frames_b[sig / p.channels] : p.frames;
    const int out_len = VL ? out_lens[sig / p.channels] : p.out_len;
    const int t_lo = max(0, blk * OB - halo);
    const int t_hi = min(n_frames - 1, blk * OB + OB - 1);
    const int nfr = t_hi - t_lo + 1;
    if constexpr (VL) {
        if (nfr <= 0) {              // entirely past this signal's end: its share of the row is padding
            float* ys = y + (int64_t)sig * p.out_len;
            for (int i = tid; i < OB * p.hop; i += NTH) {
                const int n_out = blk * OB * p.hop + i - N / 2;
                if (n_out >= out_len && n_out < p.out_len) ys[n_out] = 0.f;
            }
            return;
        }
    }
    if (tid < 256) {
        float sn, cs;
        sincospif(2.0f * (float)tid / 256.0f, &sn, &cs);
        tw256[tid] = make_float2(cs, sn);
        sincospif(2.0f * (float)tid / 512.0f, &sn, &cs);
        twp[tid] = make_float2(cs, sn);
        if (tid == 0) twp[256] = make_float2(-1.f, 0.f);
    }
    const int wl = (N - p.win) / 2;
    for (int n = tid; n < N; n += NTH) { const int k = n - wl; wpad[n] = (k >= 0 && k < p.win) ? window[k] : 0.0f; }
    const float* zs = z + (int64_t)(sig / p.channels) * p.z_stride_b + (int64_t)(sig % p.channels) * p.z_stride_c;
    for (int i = tid; i < (M + 1) * nfr; i += NTH) {
        const int k = i / nfr, f2 = i - k * nfr;
        float2 o = make_float2(0.f, 0.f);
        if (k < p.bins_in) o = *reinterpret_cast<const float2*>(zs + (int64_t)k * p.z_stride_k + (int64_t)(t_lo + f2) * p.z_stride_t);
        if (k == 0 || k == M) o.y = 0.f;
        xsb[f2 * (M + 1) + k] = o;
    }
    __syncthreads();

    const int fr = tid >> 4, c = tid & 15;
    float2 v[16];
    if (fr < nfr) {
        // Y[k] = Xe[k] + i Xo[k], k = 16 k1' + c  (pass 1 runs over the "slow" index, as in the forward transform)
        const float2* xf = xsb + fr * (M + 1);
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const int k = 16 * n1 + c;
            const float2 a = xf[k], b = xf[M - k];
            const float2 xe = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y - b.y));
            const float2 d = make_float2(0.5f * (a.x - b.x), 0.5f * (a.y + b.y));
            const float2 xo = cmul(twp[k], d);
            v[n1] = make_float2(xe.x - xo.y, xe.y + xo.x);
        }
        dft16<true>(v);
    }
    __syncthreads();                                                      // all reads of xsb done: reuse it as the transpose buffer
    float2* tbuf = xsb;
    if (fr < nfr) {
#pragma unroll
        for (int k1 = 0; k1 < 16; ++k1) tbuf[(fr * 16 + c) * kTPad + k1] = cmul(v[k1], tw256[c * k1]);
    }
    __syncthreads();
    if (fr < nfr) {
#pragma unroll
        for (int n2 = 0; n2 < 16; ++n2) v[n2] = tbuf[(fr * 16 + n2) * kTPad + c];
        dft16<true>(v);
    }
    __syncthreads();                                                      // pass-2 inputs are in registers: reuse the buffer
    float2* work = xsb;
    if (fr < nfr) {
#pragma unroll
        for (int k2 = 0; k2 < 16; ++k2) work[fr * M + c + 16 * k2] = v[k2];      // = (x[2n], x[2n+1]) * M, n = c + 16 k2
    }
    __syncthreads();

    const float* frames = reinterpret_cast<const float*>(work);
    const float scale = 2.0f * rsqrtf((float)N);
    const int p0 = blk * OB * p.hop, span = OB * p.hop;
    float* ys = y + (int64_t)sig * p.out_len;
    for (int i = tid; i < span; i += NTH) {
        const int pos = p0 + i;
        const int n_out = pos - N / 2;
        if (n_out < 0 || n_out >= p.out_len) continue;
        if constexpr (VL) {
            if (n_out >= out_len) { ys[n_out] = 0.f; continue; }
        }
        int ta = (pos - N + p.hop) / p.hop;
        if (pos - N + 1 <= 0) ta = 0;
        ta = max(ta, t_lo);
        const int tb = min(pos / p.hop, t_hi);
        float acc = 0.f, env = 0.f;
        for (int t = ta; t <= tb; ++t) {
            const int n = pos - t * p.hop;
            const float w = wpad[n];
            acc += frames[(t - t_lo) * N + n] * w;
            env += w * w;
        }
        ys[n_out] = acc * scale / env;
    }
}

template <int NF>
__global__ void __launch_bounds__(NF * 16) istft512_kernel(const float* __restrict__ z, const float* __restrict__ window,
                                                           float* __restrict__ y, const aero_istft_params p, const int OB,
                                                           const int halo) {
    istft512_block<NF, false>(z, window, y, p, OB, halo, nullptr, nullptr);
}

template <int NF>
__global__ void __launch_bounds__(NF * 16) istft512_varlen_kernel(const float* __restrict__ z, const float* __restrict__ window,
                                                                  float* __restrict__ y, const aero_istft_params p, const int OB,
                                                                  const int halo, const int32_t* __restrict__ frames_b,
                                                                  const int32_t* __restrict__ out_lens) {
    istft512_block<NF, true>(z, window, y, p, OB, halo, frames_b, out_lens);
}

static int launch_istft512(const float* z, const float* window, float* y, const int32_t* frames, const int32_t* out_lens,
                           const aero_istft_params& p, cudaStream_t st) {
    constexpr int NF = kI512;
    const int halo = 511 / p.hop;
    const int OB = NF - halo;
    const size_t smem = sizeof(float2) * ((size_t)NF * 16 * kTPad + 256 + 260) + sizeof(float) * 512;
    const int last_pos = 256 + p.out_len - 1;
    dim3 grid(last_pos / (OB * p.hop) + 1, p.n_signals);
    if (frames) {
        cudaFuncSetAttribute(istft512_varlen_kernel<NF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        istft512_varlen_kernel<NF><<<grid, NF * 16, smem, st>>>(z, window, y, p, OB, halo, frames, out_lens);
        return check_launch("aero_istft_varlen_fwd(512)");
    }
    cudaFuncSetAttribute(istft512_kernel<NF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    istft512_kernel<NF><<<grid, NF * 16, smem, st>>>(z, window, y, p, OB, halo);
    return check_launch("aero_istft_fwd(512)");
}

static int log2_exact(int n) {
    int l = 0;
    while ((1 << l) < n) ++l;
    return (1 << l) == n ? l : -1;
}

// ---------------------------------------------------------------------------------- entry points
// One check and one kernel choice per transform for the fixed-length entry point and its ragged twin; per-clip lengths
// (frame counts) select the ragged kernels and the ragged entry point's name in errors.
static int stft(const float* x, const float* window, float* z, double* stats, const int32_t* lengths,
                const aero_stft_params* p, cudaStream_t st) {
    const char* fn = stft_entry(lengths);
    AERO_REQUIRE(x && window && z && p, "%s: null argument", fn);
    const int lg = log2_exact(p->n_fft);
    AERO_REQUIRE(lg >= 6 && lg <= 12, "%s: n_fft=%d must be a power of two in [64,4096]", fn, p->n_fft);
    AERO_REQUIRE(p->win >= 1 && p->win <= p->n_fft && p->hop >= 1, "%s: bad win/hop %d/%d", fn, p->win, p->hop);
    if (lengths) {
        AERO_REQUIRE(p->flags == 0, "%s: flags must be 0", fn);
        AERO_REQUIRE(p->length % p->hop == 0 && p->frames == 1 + p->length / p->hop,
                     "%s: length=%d must be a multiple of hop and frames=%d == 1+length/hop", fn, p->length, p->frames);
    } else {
        AERO_REQUIRE((p->flags & AERO_STFT_ZERO_PAD) || p->length > p->n_fft / 2,
                     "%s: reflect padding needs length (%d) > n_fft/2", fn, p->length);
        AERO_REQUIRE(p->frames == 1 + p->length / p->hop, "%s: frames=%d != 1+length/hop", fn, p->frames);
    }
    AERO_REQUIRE(p->bins_out >= 1 && p->bins_out <= p->n_fft / 2 + 1, "%s: bins_out=%d", fn, p->bins_out);
    AERO_REQUIRE(p->n_signals >= 1 && p->channels >= 1 && p->n_signals % p->channels == 0, "%s: signals/channels", fn);
    AERO_REQUIRE(((p->z_stride_b | p->z_stride_c | p->z_stride_k | p->z_stride_t) & 1) == 0 && ((uintptr_t)z & 7) == 0,
                 "%s: output strides must keep float2 alignment", fn);
    if (lg == 9 && p->flags == 0 && p->hop % 2 == 0 && (size_t)(kF512 - 1) * p->hop * 4 <= 96 * 1024)
        return launch_stft512(x, window, z, stats, lengths, *p, st);
    switch (lg) {
        case 6: return launch_stft<6>(x, window, z, stats, lengths, *p, st);
        case 7: return launch_stft<7>(x, window, z, stats, lengths, *p, st);
        case 8: return launch_stft<8>(x, window, z, stats, lengths, *p, st);
        case 9: return launch_stft<9>(x, window, z, stats, lengths, *p, st);
        case 10: return launch_stft<10>(x, window, z, stats, lengths, *p, st);
        case 11: return launch_stft<11>(x, window, z, stats, lengths, *p, st);
        default: return launch_stft<12>(x, window, z, stats, lengths, *p, st);
    }
}

static int istft(const float* z, const float* window, float* y, const int32_t* frames, const int32_t* out_lens,
                 const aero_istft_params* p, cudaStream_t st) {
    const char* fn = istft_entry(frames);
    AERO_REQUIRE(z && window && y && p, "%s: null argument", fn);
    const int lg = log2_exact(p->n_fft);
    AERO_REQUIRE(lg >= 6 && lg <= 12, "%s: n_fft=%d must be a power of two in [64,4096]", fn, p->n_fft);
    AERO_REQUIRE(p->win >= 1 && p->win <= p->n_fft && p->hop >= 1, "%s: bad win/hop", fn);
    AERO_REQUIRE(!frames || p->flags == 0, "%s: flags must be 0", fn);
    AERO_REQUIRE(p->bins_in >= 1 && p->bins_in <= p->n_fft / 2 + 1, "%s: bins_in=%d", fn, p->bins_in);
    AERO_REQUIRE(p->out_len >= 1 && p->out_len <= p->hop * (p->frames - 1) + ((p->flags & AERO_ISTFT_RAW) ? p->n_fft : 0),
                 "%s: out_len=%d > hop*(frames-1)", fn, p->out_len);
    AERO_REQUIRE(p->n_signals >= 1 && p->channels >= 1 && p->n_signals % p->channels == 0, "%s: signals/channels", fn);
    AERO_REQUIRE(((p->z_stride_b | p->z_stride_c | p->z_stride_k | p->z_stride_t) & 1) == 0 && ((uintptr_t)z & 7) == 0,
                 "%s: input strides must keep float2 alignment", fn);
    if (lg == 9 && p->flags == 0 && kI512 - 511 / p->hop >= 8)      // tiny hops fall back to the generic kernel
        return launch_istft512(z, window, y, frames, out_lens, *p, st);
    switch (lg) {
        case 6: return launch_istft<6>(z, window, y, frames, out_lens, *p, st);
        case 7: return launch_istft<7>(z, window, y, frames, out_lens, *p, st);
        case 8: return launch_istft<8>(z, window, y, frames, out_lens, *p, st);
        case 9: return launch_istft<9>(z, window, y, frames, out_lens, *p, st);
        case 10: return launch_istft<10>(z, window, y, frames, out_lens, *p, st);
        case 11: return launch_istft<11>(z, window, y, frames, out_lens, *p, st);
        default: return launch_istft<12>(z, window, y, frames, out_lens, *p, st);
    }
}

}  // namespace aero

extern "C" int aero_stft_fwd(const float* x, const float* window, float* z, double* stats, const aero_stft_params* p,
                             aero_stream_t stream) {
    return aero::stft(x, window, z, stats, nullptr, p, (cudaStream_t)stream);
}

extern "C" int aero_istft_fwd(const float* z, const float* window, float* y, const aero_istft_params* p,
                              aero_stream_t stream) {
    return aero::istft(z, window, y, nullptr, nullptr, p, (cudaStream_t)stream);
}

extern "C" int aero_stft_varlen_fwd(const float* x, const float* window, float* z, double* stats, const int32_t* lengths,
                                    const aero_stft_params* p, aero_stream_t stream) {
    AERO_REQUIRE(lengths, "aero_stft_varlen_fwd: null argument");
    return aero::stft(x, window, z, stats, lengths, p, (cudaStream_t)stream);
}

extern "C" int aero_istft_varlen_fwd(const float* z, const float* window, float* y, const int32_t* frames,
                                     const int32_t* out_lens, const aero_istft_params* p, aero_stream_t stream) {
    AERO_REQUIRE(frames && out_lens, "aero_istft_varlen_fwd: null argument");
    return aero::istft(z, window, y, frames, out_lens, p, (cudaStream_t)stream);
}
