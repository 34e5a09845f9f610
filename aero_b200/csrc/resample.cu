// SEANet input stage (reference src/models/seanet.py:158-168), torchaudio.functional.resample, and the reflection-halo pass that feeds its reflect-padded
// convolutions (seanet.py:14-16,57-66,106-118).  See include/aero_b200.h for the contracts.
#include "common.cuh"

namespace aero {

constexpr int kStatThreads = 256;

// one CTA per clip: std of the channel mean (unbiased, two passes in fp64) -> affine[b] = {std, 0}
// VL (ragged batch, aero_seanet_input_varlen_fwd): clip b has lengths[b] valid samples in rows of p.L_in; the sums run over
// those samples only, in the order a single-clip call of that length uses.
template <bool VL>
__device__ __forceinline__ void seanet_std_block(const float* __restrict__ x, float* __restrict__ affine,
                                                 const int32_t* __restrict__ lengths, const aero_resample_params p) {
    __shared__ double red[kStatThreads / 32];
    __shared__ double mean_s;
    const int b = blockIdx.x;
    const float* xb = x + (int64_t)b * p.C * p.L_in;
    const int n = VL ? min(lengths[b], p.L_in) : p.L_in;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    auto mono = [&](int i) {
        float s = 0.f;
        for (int c = 0; c < p.C; ++c) s += xb[(int64_t)c * p.L_in + i];
        return s / (float)p.C;
    };
    auto block_sum = [&](double v) {
        v = warp_sum(v);
        if (lane == 0) red[warp] = v;
        __syncthreads();
        double t = 0.0;
        if (threadIdx.x == 0)
            for (int w = 0; w < kStatThreads / 32; ++w) t += red[w];
        __syncthreads();
        return t;                                        // valid in thread 0
    };
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += kStatThreads) s += mono(i);
    s = block_sum(s);
    if (threadIdx.x == 0) mean_s = s / n;
    __syncthreads();
    const double mean = mean_s;
    double q = 0.0;
    for (int i = threadIdx.x; i < n; i += kStatThreads) {
        const double d = (double)mono(i) - mean;
        q += d * d;
    }
    q = block_sum(q);
    if (threadIdx.x == 0) {
        affine[2 * b] = p.normalize ? (float)sqrt(q / (n - 1)) : 1.f;
        affine[2 * b + 1] = 0.f;
    }
}

__global__ void __launch_bounds__(kStatThreads) seanet_std_kernel(const float* __restrict__ x, float* __restrict__ affine,
                                                                  const aero_resample_params p) {
    seanet_std_block<false>(x, affine, nullptr, p);
}

__global__ void __launch_bounds__(kStatThreads) seanet_std_varlen_kernel(const float* __restrict__ x, float* __restrict__ affine,
                                                                         const int32_t* __restrict__ lengths,
                                                                         const aero_resample_params p) {
    seanet_std_block<true>(x, affine, lengths, p);
}

// Output sample t of one row of torchaudio.functional.resample's polyphase filter (_apply_sinc_resample_kernel): phase t % up
// of filt[up][taps] over the input samples (t / up) * orig - width + k, zero outside [0, L_in), each divided by `den` first.
__device__ __forceinline__ float polyphase_sample(const float* __restrict__ xs, const float* __restrict__ filt, int t, int L_in,
                                                  int orig, int up, int width, int taps, float den) {
    const int ph = t % up, s0 = (t / up) * orig - width;
    const float* f = filt + (int64_t)ph * taps;
    float v = 0.f;
    for (int k = 0; k < taps; ++k) {
        const int j = s0 + k;
        if (j >= 0 && j < L_in) v = fmaf(f[k], xs[j] / den, v);
    }
    return v;
}

// one thread per written (clip, frame, channel): normalise, polyphase filter, zero pad, reflect into the halo
// VL: clip b reads its own lengths[b] samples, is zero padded from hr_lengths[b] to valid_lengths[b] frames and reflected at
// that end; its frames from valid_lengths[b] + fill to the buffer's end (p.L_valid + p.halo) are written as zeros.
template <bool VL>
__device__ __forceinline__ void seanet_resample_body(const float* __restrict__ x, const float* __restrict__ filt,
                                                     const float* __restrict__ affine, float* __restrict__ x0,
                                                     const int32_t* __restrict__ lengths, const int32_t* __restrict__ hr_lengths,
                                                     const int32_t* __restrict__ valid_lengths, const aero_resample_params p) {
    const int span = VL ? p.L_valid + p.halo + p.fill : p.L_valid + 2 * p.fill;
    const int64_t n = (int64_t)p.B * span * p.C;
    const int64_t rows = (int64_t)p.L_valid + 2 * p.halo;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % p.C);
        const int64_t r = i / p.C;
        const int u = (int)(r % span) - p.fill;
        const int b = (int)(r / span);
        int t = u < 0 ? -u : u;
        float v = 0.f;
        if constexpr (VL) {
            // out of contract (a table entry past the buffer), every read stays inside the clip's row
            const int L_in = min(lengths[b], p.L_in), Lv = min(valid_lengths[b], p.L_valid);
            const int L_hr = min(hr_lengths[b], p.up == 0 ? L_in : Lv);
            if (u < Lv + p.fill) {
                if (t >= Lv) t = 2 * (Lv - 1) - t;
                if (t >= 0 && t < L_hr) {
                    const float den = p.normalize ? p.floor_ + affine[2 * b] : 1.f;
                    const float* xs = x + ((int64_t)b * p.C + c) * p.L_in;
                    v = p.up == 0 ? xs[t] / den : polyphase_sample(xs, filt, t, L_in, p.orig, p.up, p.width, p.taps, den);
                }
            }
        } else {
            if (t >= p.L_valid) t = 2 * (p.L_valid - 1) - t;
            if (t < p.L_hr) {
                const float den = p.normalize ? p.floor_ + affine[2 * b] : 1.f;
                const float* xs = x + ((int64_t)b * p.C + c) * p.L_in;
                v = p.up == 0 ? xs[t] / den : polyphase_sample(xs, filt, t, p.L_in, p.orig, p.up, p.width, p.taps, den);
            }
        }
        x0[((int64_t)b * rows + p.halo + u) * p.C + c] = v;
    }
}

__global__ void __launch_bounds__(256) seanet_resample_kernel(const float* __restrict__ x, const float* __restrict__ filt,
                                                              const float* __restrict__ affine, float* __restrict__ x0,
                                                              const aero_resample_params p) {
    seanet_resample_body<false>(x, filt, affine, x0, nullptr, nullptr, nullptr, p);
}

__global__ void __launch_bounds__(256) seanet_resample_varlen_kernel(const float* __restrict__ x, const float* __restrict__ filt,
                                                                     const float* __restrict__ affine, float* __restrict__ x0,
                                                                     const int32_t* __restrict__ lengths,
                                                                     const int32_t* __restrict__ hr_lengths,
                                                                     const int32_t* __restrict__ valid_lengths,
                                                                     const aero_resample_params p) {
    seanet_resample_body<true>(x, filt, affine, x0, lengths, hr_lengths, valid_lengths, p);
}

// torchaudio.functional.resample on rows of L_in samples: one thread per output sample
__global__ void __launch_bounds__(256) resample_kernel(const float* __restrict__ x, const float* __restrict__ filt, float* __restrict__ y,
                                                       int64_t rows, int L_in, int L_out, int orig, int up, int width, int taps) {
    const int64_t n = rows * L_out;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / L_out;
        const int t = (int)(i - r * L_out);
        y[i] = polyphase_sample(x + r * L_in, filt, t, L_in, orig, up, width, taps, 1.f);
    }
}

// VL (ragged batch, aero_reflect_act_varlen_fwd): clip b has frames[b] of the T frames; it is reflected at its own end, and its
// frames from frames[b] + halo to T + halo are written as zeros.
template <typename TI, typename TO, bool VL>
__device__ __forceinline__ void reflect_act_body(const TI* __restrict__ x, TO* __restrict__ y, const int32_t* __restrict__ frames,
                                                 int B, int T, int C, int64_t x_sb, int64_t y_sb, int halo, int act, bool rnd) {
    const int span = T + 2 * halo, cq = C / 4;
    const int64_t n = (int64_t)B * span * cq;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % cq) * 4;
        const int64_t r = i / cq;
        const int u = (int)(r % span) - halo;
        const int b = (int)(r / span);
        int t = u < 0 ? -u : u;
        if constexpr (VL) {
            const int Tb = min(frames[b], T);
            if (u >= Tb + halo) {
                st4(y + (int64_t)b * y_sb + (int64_t)u * C + c, make_float4(0.f, 0.f, 0.f, 0.f));
                continue;
            }
            if (t >= Tb) t = 2 * (Tb - 1) - t;
            t = min(max(t, 0), T - 1);           // out of contract (frames[b] <= halo): the read stays inside the clip's row
        } else {
            if (t >= T) t = 2 * (T - 1) - t;
        }
        float4 v = ld4(x + (int64_t)b * x_sb + (int64_t)t * C + c);
        if (act == AERO_ACT_LEAKY) {
            v.x = v.x > 0.f ? v.x : 0.2f * v.x; v.y = v.y > 0.f ? v.y : 0.2f * v.y;
            v.z = v.z > 0.f ? v.z : 0.2f * v.z; v.w = v.w > 0.f ? v.w : 0.2f * v.w;
        }
        if (rnd) { v.x = round_tf32_rna(v.x); v.y = round_tf32_rna(v.y); v.z = round_tf32_rna(v.z); v.w = round_tf32_rna(v.w); }
        st4(y + (int64_t)b * y_sb + (int64_t)u * C + c, v);
    }
}

template <typename TI, typename TO>
__global__ void __launch_bounds__(256) reflect_act_kernel(const TI* __restrict__ x, TO* __restrict__ y, int B, int T, int C,
                                                          int64_t x_sb, int64_t y_sb, int halo, int act, bool rnd) {
    reflect_act_body<TI, TO, false>(x, y, nullptr, B, T, C, x_sb, y_sb, halo, act, rnd);
}

template <typename TI, typename TO>
__global__ void __launch_bounds__(256) reflect_act_varlen_kernel(const TI* __restrict__ x, TO* __restrict__ y,
                                                                 const int32_t* __restrict__ frames, int B, int T, int C,
                                                                 int64_t x_sb, int64_t y_sb, int halo, int act, bool rnd) {
    reflect_act_body<TI, TO, true>(x, y, frames, B, T, C, x_sb, y_sb, halo, act, rnd);
}

__global__ void __launch_bounds__(256) reflect_act_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                              float* __restrict__ dx, int B, int T, int C, int64_t x_sb, int64_t dy_sb,
                                                              int halo, int act) {
    const int64_t n = (int64_t)B * T * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int64_t r = i / C;
        const int t = (int)(r % T), b = (int)(r / T);
        const float* d = dy + (int64_t)b * dy_sb + c;
        float g = d[(int64_t)t * C];
        if (t >= 1 && t <= halo) g += d[-(int64_t)t * C];                       // mirrored before frame 0
        const int u = 2 * (T - 1) - t;                                           // mirrored after frame T-1
        if (u >= T && u < T + halo) g += d[(int64_t)u * C];
        if (act == AERO_ACT_LEAKY && !(x[(int64_t)b * x_sb + (int64_t)t * C + c] > 0.f)) g *= 0.2f;
        dx[i] = g;
    }
}

__global__ void __launch_bounds__(256) seanet_output_kernel(const float* __restrict__ v, const float* __restrict__ x0,
                                                            const float* __restrict__ affine, const float* __restrict__ dy,
                                                            float* __restrict__ out, int B, int64_t per_clip, bool bwd) {
    const int64_t n = (int64_t)B * per_clip;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float s = affine[2 * (i / per_clip)];
        const float t = tanhf(v[i]);
        out[i] = bwd ? dy[i] * s * (1.f - t * t) : s * (t + x0[i]);
    }
}

static int grid_for(int64_t n) {
    const int64_t blocks = (n + 255) / 256;
    return (int)(blocks < 132 * 16 ? (blocks < 1 ? 1 : blocks) : 132 * 16);
}

}  // namespace aero

namespace aero {

// Both input-stage entry points: per-clip tables (all three, or none) select the ragged kernels.
static int seanet_input(const float* x, const float* filt, float* affine, float* x0, const int32_t* lengths,
                        const int32_t* hr_lengths, const int32_t* valid_lengths, const aero_resample_params* pp, cudaStream_t st) {
    const bool vl = lengths != nullptr;
    const char* fn = vl ? "aero_seanet_input_varlen_fwd" : "aero_seanet_input_fwd";
    AERO_REQUIRE(x && affine && x0 && pp && (!vl || (hr_lengths && valid_lengths)), "%s: null argument", fn);
    const aero_resample_params& p = *pp;
    AERO_REQUIRE(p.B >= 1 && p.C >= 1 && p.L_in >= 2, "%s: bad sizes (B=%d C=%d L_in=%d)", fn, p.B, p.C, p.L_in);
    AERO_REQUIRE(p.up >= 0 && (p.up == 0 || (filt && p.orig >= 1 && p.taps >= 1 && p.width >= 0)),
                 "%s: bad filter (up=%d orig=%d taps=%d)", fn, p.up, p.orig, p.taps);
    AERO_REQUIRE(p.up != 0 || p.L_hr == p.L_in, "%s: without resampling L_hr must equal L_in", fn);
    AERO_REQUIRE(p.L_hr >= 1 && p.L_valid >= p.L_hr && p.fill >= 0 && p.fill <= p.halo && p.fill < p.L_valid,
                 "%s: bad lengths (L_hr=%d L_valid=%d halo=%d fill=%d)", fn, p.L_hr, p.L_valid, p.halo, p.fill);
    if (vl) {
        seanet_std_varlen_kernel<<<p.B, kStatThreads, 0, st>>>(x, affine, lengths, p);
        int rc = check_launch("aero_seanet_input_varlen_fwd(std)");
        if (rc != AERO_OK) return rc;
        seanet_resample_varlen_kernel<<<grid_for((int64_t)p.B * (p.L_valid + p.halo + p.fill) * p.C), 256, 0, st>>>(
            x, filt, affine, x0, lengths, hr_lengths, valid_lengths, p);
        return check_launch("aero_seanet_input_varlen_fwd(resample)");
    }
    seanet_std_kernel<<<p.B, kStatThreads, 0, st>>>(x, affine, p);
    int rc = check_launch("aero_seanet_input_fwd(std)");
    if (rc != AERO_OK) return rc;
    seanet_resample_kernel<<<grid_for((int64_t)p.B * (p.L_valid + 2 * p.fill) * p.C), 256, 0, st>>>(x, filt, affine, x0, p);
    return check_launch("aero_seanet_input_fwd(resample)");
}

// Both reflection-halo entry points: `frames` (per-clip frame counts) selects the ragged kernel.
static int reflect_act(const void* x, void* y, const int32_t* frames, int32_t B, int32_t T, int32_t C, int64_t x_sb, int64_t y_sb,
                       int32_t halo, int32_t act, int32_t flags, cudaStream_t st) {
    const char* fn = frames ? "aero_reflect_act_varlen_fwd" : "aero_reflect_act_fwd";
    AERO_REQUIRE(x && y, "%s: null argument", fn);
    AERO_REQUIRE(B >= 1 && T >= 1 && C >= 4 && C % 4 == 0 && halo >= 0 && halo < T, "%s: bad sizes (B=%d T=%d C=%d halo=%d)", fn, B,
                 T, C, halo);
    AERO_REQUIRE(act == AERO_ACT_NONE || act == AERO_ACT_LEAKY, "%s: act=%d", fn, act);
    const bool a16 = flags & AERO_TG_A_F16, o16 = flags & AERO_TG_OUT_F16, rnd = (flags & AERO_TG_ROUND_TF32) && !o16;
    AERO_REQUIRE(!a16 || o16, "%s: FP16 input needs FP16 output", fn);
    const int g = grid_for((int64_t)B * (T + 2 * halo) * (C / 4));
    if (frames) {
        if (a16)
            reflect_act_varlen_kernel<__half, __half><<<g, 256, 0, st>>>(static_cast<const __half*>(x), static_cast<__half*>(y),
                                                                         frames, B, T, C, x_sb, y_sb, halo, act, false);
        else if (o16)
            reflect_act_varlen_kernel<float, __half><<<g, 256, 0, st>>>(static_cast<const float*>(x), static_cast<__half*>(y),
                                                                        frames, B, T, C, x_sb, y_sb, halo, act, false);
        else
            reflect_act_varlen_kernel<float, float><<<g, 256, 0, st>>>(static_cast<const float*>(x), static_cast<float*>(y), frames,
                                                                       B, T, C, x_sb, y_sb, halo, act, rnd);
        return check_launch(fn);
    }
    if (a16)
        reflect_act_kernel<__half, __half><<<g, 256, 0, st>>>(static_cast<const __half*>(x), static_cast<__half*>(y), B, T, C, x_sb,
                                                              y_sb, halo, act, false);
    else if (o16)
        reflect_act_kernel<float, __half><<<g, 256, 0, st>>>(static_cast<const float*>(x), static_cast<__half*>(y), B, T, C, x_sb,
                                                             y_sb, halo, act, false);
    else
        reflect_act_kernel<float, float><<<g, 256, 0, st>>>(static_cast<const float*>(x), static_cast<float*>(y), B, T, C, x_sb,
                                                            y_sb, halo, act, rnd);
    return check_launch(fn);
}

}  // namespace aero

extern "C" int aero_seanet_input_fwd(const float* x, const float* filt, float* affine, float* x0, const aero_resample_params* pp,
                                     aero_stream_t stream) {
    return aero::seanet_input(x, filt, affine, x0, nullptr, nullptr, nullptr, pp, (cudaStream_t)stream);
}

extern "C" int aero_seanet_input_varlen_fwd(const float* x, const float* filt, float* affine, float* x0, const int32_t* lengths,
                                            const int32_t* hr_lengths, const int32_t* valid_lengths, const aero_resample_params* pp,
                                            aero_stream_t stream) {
    AERO_REQUIRE(lengths, "aero_seanet_input_varlen_fwd: null argument");
    return aero::seanet_input(x, filt, affine, x0, lengths, hr_lengths, valid_lengths, pp, (cudaStream_t)stream);
}

extern "C" int aero_resample_fwd(const float* x, const float* filt, float* y, int64_t rows, int32_t L_in, int32_t L_out, int32_t orig,
                                 int32_t up, int32_t width, int32_t taps, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(x && filt && y, "aero_resample_fwd: null argument");
    AERO_REQUIRE(rows >= 1 && L_in >= 1 && L_out >= 1, "aero_resample_fwd: bad sizes (rows=%lld L_in=%d L_out=%d)", (long long)rows, L_in,
                 L_out);
    AERO_REQUIRE(orig >= 1 && up >= 1 && width >= 0 && taps >= 1, "aero_resample_fwd: bad filter (orig=%d up=%d width=%d taps=%d)", orig,
                 up, width, taps);
    AERO_REQUIRE((int64_t)L_out <= ((int64_t)L_in / orig + 1) * up, "aero_resample_fwd: L_out=%d exceeds the filter's %lld frames",
                 L_out, (long long)(((int64_t)L_in / orig + 1) * up));
    resample_kernel<<<grid_for(rows * L_out), 256, 0, (cudaStream_t)stream>>>(x, filt, y, rows, L_in, L_out, orig, up, width, taps);
    return check_launch("aero_resample_fwd");
}

extern "C" int aero_reflect_act_fwd(const void* x, void* y, int32_t B, int32_t T, int32_t C, int64_t x_sb, int64_t y_sb,
                                    int32_t halo, int32_t act, int32_t flags, aero_stream_t stream) {
    return aero::reflect_act(x, y, nullptr, B, T, C, x_sb, y_sb, halo, act, flags, (cudaStream_t)stream);
}

extern "C" int aero_reflect_act_varlen_fwd(const void* x, void* y, const int32_t* frames, int32_t B, int32_t T, int32_t C, int64_t x_sb,
                                           int64_t y_sb, int32_t halo, int32_t act, int32_t flags, aero_stream_t stream) {
    AERO_REQUIRE(frames, "aero_reflect_act_varlen_fwd: null argument");
    return aero::reflect_act(x, y, frames, B, T, C, x_sb, y_sb, halo, act, flags, (cudaStream_t)stream);
}

extern "C" int aero_reflect_act_bwd(const float* x, const float* dy, float* dx, int32_t B, int32_t T, int32_t C, int64_t x_sb, int64_t dy_sb,
                                    int32_t halo, int32_t act, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(dy && dx && (x || act == AERO_ACT_NONE), "aero_reflect_act_bwd: null argument");
    AERO_REQUIRE(B >= 1 && T >= 1 && C >= 1 && halo >= 0 && halo < T, "aero_reflect_act_bwd: bad sizes (B=%d T=%d C=%d halo=%d)", B, T, C,
                 halo);
    AERO_REQUIRE(act == AERO_ACT_NONE || act == AERO_ACT_LEAKY, "aero_reflect_act_bwd: act=%d", act);
    reflect_act_bwd_kernel<<<grid_for((int64_t)B * T * C), 256, 0, (cudaStream_t)stream>>>(x, dy, dx, B, T, C, x_sb, dy_sb, halo, act);
    return check_launch("aero_reflect_act_bwd");
}

extern "C" int aero_seanet_output_fwd(const float* v, const float* x0, const float* affine, float* y, int32_t B, int64_t per_clip,
                                      aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(v && x0 && affine && y && B >= 1 && per_clip >= 1, "aero_seanet_output_fwd: bad arguments");
    seanet_output_kernel<<<grid_for((int64_t)B * per_clip), 256, 0, (cudaStream_t)stream>>>(v, x0, affine, nullptr, y, B, per_clip, false);
    return check_launch("aero_seanet_output_fwd");
}

extern "C" int aero_seanet_output_bwd(const float* v, const float* affine, const float* dy, float* dv, int32_t B, int64_t per_clip,
                                      aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(v && affine && dy && dv && B >= 1 && per_clip >= 1, "aero_seanet_output_bwd: bad arguments");
    seanet_output_kernel<<<grid_for((int64_t)B * per_clip), 256, 0, (cudaStream_t)stream>>>(v, nullptr, affine, dy, dv, B, per_clip, true);
    return check_launch("aero_seanet_output_bwd");
}
