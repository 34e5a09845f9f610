// Radix-2 FFT device code shared by the STFT kernels (stft.cu) and the fused log-spectral distance (lsd.cu).
#pragma once
#include "common.cuh"

namespace aero {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// In-place radix-2 DIT over `nfr` frames of M = 2^LOGM complex points, input in bit-reversed
// order, twiddles tw[j] = exp(-+2 pi i j / (2M)) (table over N = 2M), sign chosen by table.
// Called by every thread of a block of NTH threads.
template <int LOGM, int NTH>
__device__ __forceinline__ void fft_inplace(float2* work, const float2* twN, int nfr) {
    constexpr int M = 1 << LOGM;
    const int total = nfr * (M / 2);
#pragma unroll 1
    for (int s = 0; s < LOGM; ++s) {
        const int half = 1 << s;
        const int tw_step = M >> s;          // N / (2*half) = 2M / (2*half)
        for (int i = threadIdx.x; i < total; i += NTH) {
            const int fr = i / (M / 2), j = i - fr * (M / 2);
            const int pos = j & (half - 1);
            const int i0 = ((j >> s) << (s + 1)) + pos;
            float2* w = work + fr * M;
            const float2 a = w[i0];
            const float2 b = cmul(w[i0 + half], twN[pos * tw_step]);
            w[i0] = make_float2(a.x + b.x, a.y + b.y);
            w[i0 + half] = make_float2(a.x - b.x, a.y - b.y);
        }
        __syncthreads();
    }
}

}  // namespace aero
