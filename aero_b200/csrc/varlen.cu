// Ragged batches (clips of different lengths in one forward; see include/aero_b200.h, "Ragged batches").
//
// Clip b occupies the first frames[b] frames of the usual channels-last [B][F][T][C] tensors; the rest are padding.  The
// passes here keep the padding out of every result:
//   aero_frame_mask_fwd         writes zeros on the padded frames of a tensor that a time-coupled convolution reads next;
//   aero_masked_stats_fwd       GroupNorm statistics over the valid frames only (the tap-GEMM STATS epilogue would count all);
//   aero_sample_norm_varlen_fwd the input standardisation with each clip's own value count;
//   aero_gather_rows_fwd        row gather by an index table: the BiLSTM framing of each clip (its own sequence length,
//                               windows and reassembly crop) onto the windowed layout of aero_lstm_rec_fwd.
// All are HBM-bound and small next to the GEMMs.
#include "common.cuh"

namespace aero {

// ------------------------------------------------------------------------- frame mask
template <typename T>
__global__ void __launch_bounds__(256) frame_mask_kernel(T* __restrict__ x, const int32_t* __restrict__ frames, int F, int Tm,
                                                         int C) {
    const int bf = blockIdx.y;
    const int tb = frames[bf / F];
    if (tb >= Tm) return;
    T* row = x + ((int64_t)bf * Tm + tb) * C;
    const int64_t n = (int64_t)(Tm - tb) * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        row[i] = T(0.f);
}

// ------------------------------------------------------------------------- masked GroupNorm statistics
// One slot (scope 1: (b, group); scope 2: row (b, f)) is split over gridDim.x CTAs; each CTA adds its partial sums, already
// scaled by Tm / frames[b], so that aero_norm_act_fwd's count over all Tm frames yields the moments of the valid frames.
template <typename TI>
__global__ void __launch_bounds__(256) masked_stats_kernel(const TI* __restrict__ x, double* __restrict__ stats,
                                                           const int32_t* __restrict__ frames, int F, int Tm, int C,
                                                           int groups, int scope) {
    const int slot = blockIdx.y;
    int b, f0, nf, c0, cw;
    if (scope == 1) { b = slot / groups; f0 = 0; nf = F; cw = C / groups; c0 = (slot % groups) * cw; }
    else { b = slot / F; f0 = slot % F; nf = 1; c0 = 0; cw = C; }
    const int tb = min(frames[b], Tm);
    const int64_t per_f = (int64_t)tb * cw;
    const int64_t n = per_f * nf;
    double s = 0.0, q = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int f = (int)(i / per_f);
        const int64_t r = i - f * per_f;
        const int t = (int)(r / cw), c = (int)(r - (int64_t)t * cw);
        const double v = (double)ldf(x + (((int64_t)b * F + f0 + f) * Tm + t) * C + c0 + c);
        s += v;
        q += v * v;
    }
    __shared__ double red[2][8];
    s = warp_sum(s);
    q = warp_sum(q);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s; red[1][threadIdx.x >> 5] = q; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, c = 0;
        for (int w = 0; w < 8; ++w) { a += red[0][w]; c += red[1][w]; }
        const double k = (double)Tm / (double)max(tb, 1);
        atomicAdd(&stats[2 * slot], a * k);
        atomicAdd(&stats[2 * slot + 1], c * k);
    }
}

// ------------------------------------------------------------------------- per-clip sample norm
// aero_sample_norm_fwd with count = per_frame * frames[b] (reference aero.py:462-464 on the clip alone)
__global__ void __launch_bounds__(256) sample_norm_varlen_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                                                 float* __restrict__ y, float* __restrict__ samp_affine,
                                                                 const int32_t* __restrict__ frames, int64_t per_frame,
                                                                 int64_t extent, int rnd) {
    const int b = blockIdx.y;
    __shared__ float s_mean, s_inv;
    if (threadIdx.x == 0) {
        const double n = (double)(per_frame * frames[b]);
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
    const float* xb = x + (int64_t)b * extent;
    float* yb = y + (int64_t)b * extent;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < extent; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = (xb[i] - mean) * inv;
        yb[i] = rnd ? round_tf32_rna(v) : v;
    }
}

// ------------------------------------------------------------------------- row gather
// dst[i][c] = src[idx[i][part]][c] with part = c / (width / parts); idx < 0 takes fill[c] (zero when fill is null)
template <typename T>
__global__ void __launch_bounds__(256) gather_rows_kernel(const T* __restrict__ src, T* __restrict__ dst,
                                                          const int32_t* __restrict__ idx, const float* __restrict__ fill,
                                                          int64_t n_rows, int width, int parts) {
    const int pw = width / parts;
    const int64_t n = n_rows * width;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / width;
        const int c = (int)(i - r * width);
        const int j = idx[r * parts + c / pw];
        dst[i] = j >= 0 ? src[(int64_t)j * width + c] : T(fill ? fill[c] : 0.f);
    }
}

static int grid_for(int64_t n, int64_t cap) {
    const int64_t g = (n + 255) / 256;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace aero

extern "C" int aero_frame_mask_fwd(void* x, const int32_t* frames, int32_t B, int32_t F, int32_t T, int32_t C, int32_t flags,
                                   aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && frames, "aero_frame_mask_fwd: null argument");
    AERO_REQUIRE(B >= 1 && F >= 1 && T >= 1 && C >= 1 && (int64_t)B * F <= 65535, "aero_frame_mask_fwd: bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(grid_for((int64_t)T * C, 64), B * F);
    if (flags & AERO_TG_OUT_F16) frame_mask_kernel<__half><<<grid, 256, 0, st>>>(static_cast<__half*>(x), frames, F, T, C);
    else frame_mask_kernel<float><<<grid, 256, 0, st>>>(static_cast<float*>(x), frames, F, T, C);
    return check_launch("aero_frame_mask_fwd");
}

extern "C" int aero_masked_stats_fwd(const void* x, double* stats, const int32_t* frames, int32_t B, int32_t F, int32_t T,
                                     int32_t C, int32_t groups, int32_t scope, int32_t flags, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && stats && frames, "aero_masked_stats_fwd: null argument");
    AERO_REQUIRE(scope == 1 || scope == 2, "aero_masked_stats_fwd: scope %d (1 or 2)", scope);
    AERO_REQUIRE(B >= 1 && F >= 1 && T >= 1 && C >= 1 && groups >= 1 && C % groups == 0, "aero_masked_stats_fwd: bad sizes");
    const int slots = scope == 1 ? B * groups : B * F;
    AERO_REQUIRE(slots <= 65535, "aero_masked_stats_fwd: %d slots", slots);
    const int64_t per_slot = scope == 1 ? (int64_t)F * T * (C / groups) : (int64_t)T * C;
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(grid_for(per_slot / 8, 128), slots);        // ~8 values per thread
    if (flags & AERO_TG_A_F16)
        masked_stats_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half*>(x), stats, frames, F, T, C, groups, scope);
    else
        masked_stats_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float*>(x), stats, frames, F, T, C, groups, scope);
    return check_launch("aero_masked_stats_fwd");
}

extern "C" int aero_sample_norm_varlen_fwd(const float* x, const double* stats, float* y, float* samp_affine,
                                           const int32_t* frames, int32_t B, int64_t per_frame, int64_t extent,
                                           int32_t round_tf32, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && stats && y && frames, "aero_sample_norm_varlen_fwd: null argument");
    AERO_REQUIRE(B >= 1 && B <= 65535 && per_frame >= 1 && extent >= 1, "aero_sample_norm_varlen_fwd: bad sizes");
    dim3 grid(grid_for(extent, 64), B);
    sample_norm_varlen_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, stats, y, samp_affine, frames, per_frame, extent,
                                                                       round_tf32);
    return check_launch("aero_sample_norm_varlen_fwd");
}

extern "C" int aero_gather_rows_fwd(const void* src, void* dst, const int32_t* idx, const float* fill, int64_t n_rows,
                                    int32_t width, int32_t parts, int32_t flags, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(src && dst && idx, "aero_gather_rows_fwd: null argument");
    AERO_REQUIRE(n_rows >= 1 && width >= 1 && parts >= 1 && width % parts == 0, "aero_gather_rows_fwd: bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = grid_for(n_rows * width, 132 * 16);
    if (flags & AERO_TG_A_F16)
        gather_rows_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half*>(src), static_cast<__half*>(dst), idx, fill,
                                                         n_rows, width, parts);
    else
        gather_rows_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float*>(src), static_cast<float*>(dst), idx, fill,
                                                        n_rows, width, parts);
    return check_launch("aero_gather_rows_fwd");
}
