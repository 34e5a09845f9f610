// Log-spectral distance on the GPU (reference src/metrics.py:37-70, `get_lsd` with STFTMag(2048, 512)):
//   LSD = mean_{b,t} sqrt( mean_f ( log10 max(|S_ref|^2, 1e-8) - log10 max(|S_est|^2, 1e-8) )^2 )
// Inputs are the *normalized* spectrograms produced by aero_stft_fwd (x n_fft^-1/2), so |S|^2 = n_fft |z|^2.
// One CTA per (b, t) column; fp64 accumulation of the per-column distances into out[0] (sum) -- the caller divides
// by B * frames.  HBM-bound: reads both spectrograms once.
#include "common.cuh"
#include "fft.cuh"

namespace aero {

__global__ void __launch_bounds__(256) lsd_kernel(const float2* __restrict__ zr, const float2* __restrict__ ze,
                                                  double* __restrict__ out, int bins, int frames, float n_fft) {
    const int t = blockIdx.x, b = blockIdx.y;
    const float2* pr = zr + ((int64_t)b * bins) * frames + t;
    const float2* pe = ze + ((int64_t)b * bins) * frames + t;
    float acc = 0.f;
    for (int f = threadIdx.x; f < bins; f += 256) {
        const float2 a = pr[(int64_t)f * frames], c = pe[(int64_t)f * frames];
        const float sp = log10f(fmaxf(n_fft * (a.x * a.x + a.y * a.y), 1e-8f));
        const float st = log10f(fmaxf(n_fft * (c.x * c.x + c.y * c.y), 1e-8f));
        acc += (sp - st) * (sp - st);
    }
    __shared__ float red[8];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += red[w];
        atomicAdd(out, (double)sqrtf(s / (float)bins));
    }
}

// ---------------------------------------------------------------------------------- ragged, fused (aero_lsd_varlen_fwd)
// Rows of different lengths, one LSD per file.  Pass 1 (lsd_frames_kernel): a CTA owns kLsdFrames consecutive frames of one
// row, builds the windowed frames of both the reference and the estimate straight from the waveforms (reflect padding at the
// row's own ends), runs the 2 * kLsdFrames real 2048-point transforms as 1024-point complex FFTs in shared memory and writes
// one fp32 distance per frame.  Pass 2 (lsd_file_mean_kernel): one CTA per file sums its frames in fp64 in a fixed order.
// No spectrogram touches HBM and no floating-point atomics: a file's value depends on its own samples only, bit for bit.
constexpr int kLsdThreads = 256;
constexpr int kLsdFrames = 4;                    // frames per CTA; 2 * 4 transforms of 1024 complex points = 64 KB
constexpr int kLsdLogM = 10, kLsdM = 1 << kLsdLogM, kLsdN = 2 * kLsdM, kLsdHop = 512;
constexpr int kLsdBins = kLsdM + 1;
constexpr size_t kLsdSmem = sizeof(float2) * (2 * kLsdFrames * kLsdM + kLsdM);

__global__ void __launch_bounds__(kLsdThreads) lsd_frames_kernel(const float* __restrict__ ref, const float* __restrict__ est,
                                                                 const int32_t* __restrict__ lengths,
                                                                 const int32_t* __restrict__ row_frame_off, int L_max,
                                                                 float* __restrict__ frame_lsd) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* work = reinterpret_cast<float2*>(smem_raw);                 // [2 * kLsdFrames][M]: transform 2 fr + s, s = 0 ref, 1 est
    float2* twN = work + 2 * kLsdFrames * kLsdM;                        // [M] exp(-2 pi i j / N)
    __shared__ float red[kLsdFrames][kLsdThreads / 32];

    const int row = blockIdx.y, tid = threadIdx.x;
    const int t0 = blockIdx.x * kLsdFrames;
    const int off = row_frame_off[row];
    const int nfr = min(kLsdFrames, row_frame_off[row + 1] - off - t0);
    if (nfr <= 0) return;
    const int L = max(1, min(lengths[row], L_max));

    for (int j = tid; j < kLsdM; j += kLsdThreads) {
        float s, c;
        sincospif(2.0f * (float)j / (float)kLsdN, &s, &c);
        twN[j] = make_float2(c, -s);
    }
    // windowed frames (periodic Hann), even/odd samples packed into one complex point, bit-reversed placement
    const float* xr = ref + (int64_t)row * L_max;
    const float* xe = est + (int64_t)row * L_max;
    for (int i = tid; i < 2 * nfr * kLsdM; i += kLsdThreads) {
        const int q = i >> kLsdLogM, n = i & (kLsdM - 1);
        const float* x = (q & 1) ? xe : xr;
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int m = 2 * n + e;                                    // sample of the frame, 0 .. N-1
            int src = (t0 + (q >> 1)) * kLsdHop - kLsdN / 2 + m;
            if (src < 0) src = -src;
            if (src >= L) src = 2 * (L - 1) - src;
            src = min(max(src, 0), L - 1);                              // only out-of-contract lengths (L <= N/2) need this
            v[e] = x[src] * (0.5f - 0.5f * cospif((float)m / (float)(kLsdN / 2)));
        }
        work[q * kLsdM + (__brev((unsigned)n) >> (32 - kLsdLogM))] = make_float2(v[0], v[1]);
    }
    __syncthreads();
    fft_inplace<kLsdLogM, kLsdThreads>(work, twN, 2 * nfr);

    // split post-pass X[k] = Xe[k] + w^k Xo[k], X[M-k] = conj(Xe[k] - w^k Xo[k]) for both signals; bins k and M-k per step
    float acc[kLsdFrames];
#pragma unroll
    for (int fr = 0; fr < kLsdFrames; ++fr) {
        acc[fr] = 0.f;
        if (fr >= nfr) continue;
        for (int k = tid; k <= kLsdM / 2; k += kLsdThreads) {
            float lg[2][2];                                             // [signal][bin k, bin M-k]: log10 max(|X|^2, 1e-8)
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                const float2* z = work + (2 * fr + s) * kLsdM;
                const float2 a = z[k], bq = z[(kLsdM - k) & (kLsdM - 1)];
                const float2 ev = make_float2(0.5f * (a.x + bq.x), 0.5f * (a.y - bq.y));
                const float2 d = make_float2(0.5f * (a.x - bq.x), 0.5f * (a.y + bq.y));
                const float2 t = cmul(twN[k], make_float2(d.y, -d.x));
                const float2 lo = make_float2(ev.x + t.x, ev.y + t.y), hi = make_float2(ev.x - t.x, ev.y - t.y);
                lg[s][0] = log10f(fmaxf(lo.x * lo.x + lo.y * lo.y, 1e-8f));
                lg[s][1] = log10f(fmaxf(hi.x * hi.x + hi.y * hi.y, 1e-8f));
            }
            const float d0 = lg[0][0] - lg[1][0], d1 = lg[0][1] - lg[1][1];
            acc[fr] += d0 * d0;
            if (k != kLsdM / 2) acc[fr] += d1 * d1;                     // k = M/2 is its own mirror
        }
    }
#pragma unroll
    for (int fr = 0; fr < kLsdFrames; ++fr) {
        const float w = warp_sum(acc[fr]);
        if ((tid & 31) == 0) red[fr][tid >> 5] = w;
    }
    __syncthreads();
    if (tid < nfr) {
        float s = 0.f;
        for (int w = 0; w < kLsdThreads / 32; ++w) s += red[tid][w];
        frame_lsd[off + t0 + tid] = sqrtf(s / (float)kLsdBins);
    }
}

// File f: the mean of the frames of its rows (rows in order, frames in order).  Thread t sums the file's frames j with
// j % kLsdThreads == t, so the order depends on the file's own frame sequence only, not on where its rows sit.
__global__ void __launch_bounds__(kLsdThreads) lsd_file_mean_kernel(const float* __restrict__ frame_lsd,
                                                                    const int32_t* __restrict__ row_file,
                                                                    const int32_t* __restrict__ row_frame_off, int rows,
                                                                    float* __restrict__ out) {
    const int f = blockIdx.x, tid = threadIdx.x;
    double acc = 0.0;
    int seen = 0;                                                       // frames of this file in the rows before r
    for (int r = 0; r < rows; ++r) {
        if (row_file[r] != f) continue;
        const int off = row_frame_off[r], n = row_frame_off[r + 1] - off;
        for (int i = (tid - seen % kLsdThreads + kLsdThreads) % kLsdThreads; i < n; i += kLsdThreads) acc += (double)frame_lsd[off + i];
        seen += n;
    }
    __shared__ double red[kLsdThreads / 32];
    acc = warp_sum(acc);
    if ((tid & 31) == 0) red[tid >> 5] = acc;
    __syncthreads();
    if (tid == 0) {
        double s = 0.0;
        for (int w = 0; w < kLsdThreads / 32; ++w) s += red[w];
        out[f] = (float)(s / (double)seen);
    }
}

}  // namespace aero

extern "C" int aero_lsd_varlen_fwd(const float* ref, const float* est, int32_t rows, int32_t L_max, const int32_t* lengths,
                                   const int32_t* row_file, const int32_t* row_frame_off, int32_t max_frames, int32_t n_files,
                                   float* frame_lsd, float* out, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(ref && est && lengths && row_file && row_frame_off && frame_lsd && out, "aero_lsd_varlen_fwd: null argument");
    AERO_REQUIRE(rows >= 1 && rows <= 65535, "aero_lsd_varlen_fwd: rows=%d must lie in [1, 65535]", rows);
    AERO_REQUIRE(L_max > kLsdN / 2, "aero_lsd_varlen_fwd: L_max=%d must exceed n_fft/2 (%d)", L_max, kLsdN / 2);
    AERO_REQUIRE(max_frames >= 1 && max_frames <= 1 + L_max / kLsdHop, "aero_lsd_varlen_fwd: max_frames=%d for L_max=%d",
                 max_frames, L_max);
    AERO_REQUIRE(n_files >= 1, "aero_lsd_varlen_fwd: n_files=%d", n_files);
    const cudaStream_t st = (cudaStream_t)stream;
    cudaFuncSetAttribute(lsd_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLsdSmem);
    lsd_frames_kernel<<<dim3(cdiv(max_frames, kLsdFrames), rows), kLsdThreads, kLsdSmem, st>>>(ref, est, lengths, row_frame_off,
                                                                                               L_max, frame_lsd);
    int rc = check_launch("aero_lsd_varlen_fwd(frames)");
    if (rc != AERO_OK) return rc;
    lsd_file_mean_kernel<<<n_files, kLsdThreads, 0, st>>>(frame_lsd, row_file, row_frame_off, rows, out);
    return check_launch("aero_lsd_varlen_fwd(files)");
}

extern "C" int aero_lsd_fwd(const float* z_ref, const float* z_est, double* out_sum, int32_t B, int32_t bins, int32_t frames,
                            int32_t n_fft, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(z_ref && z_est && out_sum && B >= 1 && bins >= 1 && frames >= 1 && n_fft >= 2, "aero_lsd_fwd: bad argument");
    AERO_REQUIRE(B <= 65535, "aero_lsd_fwd: batch too large");
    dim3 grid(frames, B);
    lsd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float2*>(z_ref), reinterpret_cast<const float2*>(z_est),
                                                      out_sum, bins, frames, (float)n_fft);
    return check_launch("aero_lsd_fwd");
}
