// HiFi-GAN multi-period discriminator (reference src/models/discriminators.py:89-147): the HBM-bound passes around its tap-GEMMs.
// Period fold (reflect pad to a multiple of the period + [T/p, p] view) and activation repack (LeakyReLU + the segment layout of
// the next layer), with their adjoints.  See include/aero_b200.h for the contracts and DESIGN.md, "Multi-period discriminator".
#include "common.cuh"

namespace aero {

static int mpd_grid(int64_t n) {
    const int64_t blocks = (n + 255) / 256;
    return (int)(blocks < 132 * 16 ? (blocks < 1 ? 1 : blocks) : 132 * 16);
}

// y[(b*P + w)*seg + u] = xp(b, (u - halo)*P + w) for halo <= u < halo + H, 0 elsewhere; xp = x reflect-padded to H*P samples
__global__ void __launch_bounds__(256) mpd_fold_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int T, int P, int H,
                                                       int seg, int halo) {
    const int64_t n = (int64_t)B * P * seg;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int u = (int)(i % seg);
        const int64_t s = i / seg;
        const int w = (int)(s % P), b = (int)(s / P);
        const int h = u - halo;
        float v = 0.f;
        if (h >= 0 && h < H) {
            int t = h * P + w;
            if (t >= T) t = 2 * (T - 1) - t;                                  // reflection of the last sample
            v = x[(int64_t)b * T + t];
        }
        y[i] = v;
    }
}

// dx(b, t) = dy at the fold position of t, plus dy at the position of its mirror image t' = 2(T-1) - t when t' lies in the padding
__global__ void __launch_bounds__(256) mpd_fold_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int B, int T, int P,
                                                           int H, int seg, int halo) {
    const int64_t n = (int64_t)B * T;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int t = (int)(i % T), b = (int)(i / T);
        const float* d = dy + (int64_t)b * P * seg + halo;
        float g = d[(int64_t)(t % P) * seg + t / P];
        const int tm = 2 * (T - 1) - t;
        if (tm >= T && tm < H * P) g += d[(int64_t)(tm % P) * seg + tm / P];
        dx[i] = g;
    }
}

// y[(s*seg + u)*C + c] = leaky(x[(s*rows_in + u - halo)*C + c]) for halo <= u < halo + H, 0 elsewhere (4 channels per thread)
__global__ void __launch_bounds__(256) mpd_repack_kernel(const float* __restrict__ x, float* __restrict__ y, int S, int H, int C4,
                                                         int rows_in, int seg, int halo, float slope) {
    const int64_t n = (int64_t)S * seg * C4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        const int64_t r = i / C4;
        const int u = (int)(r % seg);
        const int64_t s = r / seg;
        const int h = u - halo;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (h >= 0 && h < H) {
            v = reinterpret_cast<const float4*>(x)[(s * rows_in + h) * C4 + c4];
            v.x = v.x > 0.f ? v.x : v.x * slope;
            v.y = v.y > 0.f ? v.y : v.y * slope;
            v.z = v.z > 0.f ? v.z : v.z * slope;
            v.w = v.w > 0.f ? v.w : v.w * slope;
        }
        reinterpret_cast<float4*>(y)[i] = v;
    }
}

// dx[(s*rows_in + r)*C + c] = dy[(s*seg + halo + r)*C + c] * leaky'(x) for r < H, 0 for the rows r >= H no output frame owns
__global__ void __launch_bounds__(256) mpd_repack_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                             float* __restrict__ dx, int S, int H, int C4, int rows_in, int seg, int halo,
                                                             float slope) {
    const int64_t n = (int64_t)S * rows_in * C4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        const int64_t r = i / C4;
        const int h = (int)(r % rows_in);
        const int64_t s = r / rows_in;
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
        if (h < H) {
            g = reinterpret_cast<const float4*>(dy)[(s * seg + halo + h) * C4 + c4];
            const float4 v = reinterpret_cast<const float4*>(x)[i];
            if (!(v.x > 0.f)) g.x *= slope;
            if (!(v.y > 0.f)) g.y *= slope;
            if (!(v.z > 0.f)) g.z *= slope;
            if (!(v.w > 0.f)) g.w *= slope;
        }
        reinterpret_cast<float4*>(dx)[i] = g;
    }
}

static bool fold_ok(int B, int T, int P, int H, int seg, int halo) {
    return B >= 1 && T >= 1 && P >= 1 && H >= 1 && (int64_t)H * P >= T && (int64_t)H * P - T < T && (int64_t)(H - 1) * P < T &&
           halo >= 0 && halo + H <= seg;
}

static bool repack_ok(const void* a, const void* b, int S, int H, int C, int rows_in, int seg, int halo) {
    auto al16 = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
    return al16(a) && al16(b) && S >= 1 && H >= 1 && C >= 4 && C % 4 == 0 && rows_in >= H && halo >= 0 && halo + H <= seg;
}

}  // namespace aero

extern "C" int aero_mpd_fold_fwd(const float* x, float* y, int32_t B, int32_t T, int32_t period, int32_t H, int32_t seg, int32_t halo,
                                 aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && y, "aero_mpd_fold_fwd: null argument");
    AERO_REQUIRE(fold_ok(B, T, period, H, seg, halo), "aero_mpd_fold_fwd: bad sizes (B=%d T=%d period=%d H=%d seg=%d halo=%d)", B, T,
                 period, H, seg, halo);
    mpd_fold_kernel<<<mpd_grid((int64_t)B * period * seg), 256, 0, (cudaStream_t)stream>>>(x, y, B, T, period, H, seg, halo);
    return check_launch("aero_mpd_fold_fwd");
}

extern "C" int aero_mpd_fold_bwd(const float* dy, float* dx, int32_t B, int32_t T, int32_t period, int32_t H, int32_t seg, int32_t halo,
                                 aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(dy && dx, "aero_mpd_fold_bwd: null argument");
    AERO_REQUIRE(fold_ok(B, T, period, H, seg, halo), "aero_mpd_fold_bwd: bad sizes (B=%d T=%d period=%d H=%d seg=%d halo=%d)", B, T,
                 period, H, seg, halo);
    mpd_fold_bwd_kernel<<<mpd_grid((int64_t)B * T), 256, 0, (cudaStream_t)stream>>>(dy, dx, B, T, period, H, seg, halo);
    return check_launch("aero_mpd_fold_bwd");
}

extern "C" int aero_mpd_repack_fwd(const float* x, float* y, int32_t S, int32_t H, int32_t C, int32_t rows_in, int32_t seg, int32_t halo,
                                   float slope, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && y, "aero_mpd_repack_fwd: null argument");
    AERO_REQUIRE(repack_ok(x, y, S, H, C, rows_in, seg, halo),
                 "aero_mpd_repack_fwd: bad sizes or alignment (S=%d H=%d C=%d rows_in=%d seg=%d halo=%d)", S, H, C, rows_in, seg, halo);
    mpd_repack_kernel<<<mpd_grid((int64_t)S * seg * (C / 4)), 256, 0, (cudaStream_t)stream>>>(x, y, S, H, C / 4, rows_in, seg, halo,
                                                                                              slope);
    return check_launch("aero_mpd_repack_fwd");
}

extern "C" int aero_mpd_repack_bwd(const float* x, const float* dy, float* dx, int32_t S, int32_t H, int32_t C, int32_t rows_in,
                                   int32_t seg, int32_t halo, float slope, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && dy && dx, "aero_mpd_repack_bwd: null argument");
    AERO_REQUIRE(repack_ok(x, dy, S, H, C, rows_in, seg, halo) && ((uintptr_t)dx & 15) == 0,
                 "aero_mpd_repack_bwd: bad sizes or alignment (S=%d H=%d C=%d rows_in=%d seg=%d halo=%d)", S, H, C, rows_in, seg, halo);
    mpd_repack_bwd_kernel<<<mpd_grid((int64_t)S * rows_in * (C / 4)), 256, 0, (cudaStream_t)stream>>>(x, dy, dx, S, H, C / 4, rows_in,
                                                                                                       seg, halo, slope);
    return check_launch("aero_mpd_repack_bwd");
}
