// Multi-resolution STFT loss, forward reductions (SURVEY.md section 8f rank 2; reference src/models/stft_loss.py:11-27,30-63):
// for one resolution, with mag = sqrt(max(re^2 + im^2, 1e-7)) of the un-normalised STFTs of x (estimate) and y (target),
//   sums[0] += sum (mag_y - mag_x)^2      sums[1] += sum mag_y^2      sums[2] += sum |log mag_y - log mag_x|
// so that spectral convergence = sqrt(sums[0] / sums[1]) and the log-magnitude L1 = sums[2] / (B * frames * bins).
// Inputs are the *normalised* spectrograms written by aero_stft_fwd (x n_fft^-1/2): re^2 + im^2 = n_fft |z|^2.
// HBM-bound: both spectrograms are read once; fp32 per-thread partials, fp64 across the grid.
#include "common.cuh"

namespace aero {

__global__ void __launch_bounds__(256) stft_loss_kernel(const float2* __restrict__ zx, const float2* __restrict__ zy,
                                                        double* __restrict__ sums, int64_t n, float n_fft) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float2 a = zx[i], c = zy[i];
        const float px = fmaxf(n_fft * (a.x * a.x + a.y * a.y), 1e-7f), py = fmaxf(n_fft * (c.x * c.x + c.y * c.y), 1e-7f);
        const float mx = sqrtf(px), my = sqrtf(py);
        s0 += (my - mx) * (my - mx);
        s1 += py;
        s2 += 0.5f * fabsf(logf(py) - logf(px));                  // log mag = log(power) / 2
    }
    __shared__ float red[8][3];
    s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5][0] = s0; red[threadIdx.x >> 5][1] = s1; red[threadIdx.x >> 5][2] = s2; }
    __syncthreads();
    if (threadIdx.x < 3) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += (double)red[w][threadIdx.x];
        atomicAdd(sums + threadIdx.x, t);
    }
}

// Backward: gradient of  c_sc * sqrt(S0 / S1) + c_mag * S2 / n  with respect to the NORMALISED spectrogram of the estimate, written
// with the interior bins halved (G~), i.e. ready for aero_istft_fwd in AERO_ISTFT_RAW mode, whose output is then the gradient of the
// reflect-padded waveform.   d mag_x / d z' = n_fft * z' / mag_x  (zero where the 1e-7 clamp is active).
__global__ void __launch_bounds__(256) stft_loss_bwd_kernel(const float2* __restrict__ zx, const float2* __restrict__ zy,
                                                            const double* __restrict__ sums, float2* __restrict__ gz, int64_t n, float n_fft,
                                                            int bins, int frames, float c_sc, float c_mag) {
    const double s0 = sums[0], s1 = sums[1];
    const float k_sc = (s0 > 0.0 && s1 > 0.0) ? c_sc / (float)sqrt(s0 * s1) : 0.f;      // d sqrt(S0/S1) / d mag_x = -(my - mx) / sqrt(S0 S1)
    const float k_mag = c_mag / (float)n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float2 a = zx[i], c = zy[i];
        const float pxr = n_fft * (a.x * a.x + a.y * a.y);
        const float px = fmaxf(pxr, 1e-7f), py = fmaxf(n_fft * (c.x * c.x + c.y * c.y), 1e-7f);
        const float mx = sqrtf(px), my = sqrtf(py);
        float2 g = make_float2(0.f, 0.f);
        if (pxr > 1e-7f) {
            const float dl = logf(py) - logf(px);
            const float dmx = -k_sc * (my - mx) - k_mag * (dl > 0.f ? 1.f : (dl < 0.f ? -1.f : 0.f)) / mx;
            const int k = (int)((i / frames) % bins);
            const float half = (k == 0 || k == bins - 1) ? 1.0f : 0.5f;
            const float f = dmx * n_fft / mx * half;
            g = make_float2(f * a.x, f * a.y);
        }
        gz[i] = g;
    }
}

}  // namespace aero

extern "C" int aero_stft_loss_bwd(const float* z_est, const float* z_ref, const double* sums, float* g_est, int32_t B, int32_t bins,
                                  int32_t frames, int32_t n_fft, float c_sc, float c_mag, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(z_est && z_ref && sums && g_est && B >= 1 && bins == n_fft / 2 + 1 && frames >= 1, "aero_stft_loss_bwd: bad argument");
    const int64_t n = (int64_t)B * bins * frames;
    int blocks = (int)((n + 256 * 8 - 1) / (256 * 8));
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    stft_loss_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float2*>(z_est), reinterpret_cast<const float2*>(z_ref), sums,
                                                                  reinterpret_cast<float2*>(g_est), n, (float)n_fft, bins, frames, c_sc, c_mag);
    return check_launch("aero_stft_loss_bwd");
}

extern "C" int aero_stft_loss_fwd(const float* z_est, const float* z_ref, double* sums, int32_t B, int32_t bins, int32_t frames,
                                  int32_t n_fft, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(z_est && z_ref && sums && B >= 1 && bins >= 1 && frames >= 1 && n_fft >= 2, "aero_stft_loss_fwd: bad argument");
    const int64_t n = (int64_t)B * bins * frames;
    int blocks = (int)((n + 256 * 8 - 1) / (256 * 8));
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    stft_loss_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float2*>(z_est), reinterpret_cast<const float2*>(z_ref),
                                                              sums, n, (float)n_fft);
    return check_launch("aero_stft_loss_fwd");
}
