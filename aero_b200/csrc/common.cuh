// Shared helpers for libaero_b200 (sm_90a).  No torch / ATen types anywhere in csrc/.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/aero_b200.h"

namespace aero {

void set_error(const char* fmt, ...);
int check_launch(const char* what);   // bumps the launch counter, returns AERO_OK / AERO_ERR_LAUNCH

#define AERO_REQUIRE(cond, ...)                         \
    do {                                                \
        if (!(cond)) {                                  \
            aero::set_error(__VA_ARGS__);               \
            return AERO_ERR_INVALID;                    \
        }                                               \
    } while (0)

__device__ __forceinline__ float gelu_exact(float x) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float leaky_f(float x) { return x > 0.f ? x : 0.2f * x; }   // nn.LeakyReLU(0.2)

// Round to TF32 (10-bit mantissa), nearest with ties away from zero -- the result of cvt.rna.tf32.f32 for every finite input,
// in two integer instructions (ptxas expands the cvt into ~5 with Inf/NaN special-casing; Inf and NaN also survive this form:
// their low 13 mantissa bits are simply cleared).  Matches aero_b200.engine.tf32_round on the host bit for bit.
__device__ __forceinline__ float round_tf32_rna(float x) {
    return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}

// ---- activation storage types.  Tensors that feed a tensor-core GEMM are stored either as fp32 rounded to TF32 or as
// FP16 (same 10-bit mantissa, half the bytes, twice the tensor-core rate); arithmetic between loads and stores is fp32.
// FP16 stores saturate to +-65504 instead of producing Inf.
__device__ __forceinline__ float ldf(const float* p) { return *p; }
__device__ __forceinline__ float ldf(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ void stf(float* p, float v) { *p = v; }
// two fp32 -> packed FP16 pair, round-to-nearest-even, saturating at +-65504 (one F2FP.SATFINITE)
__device__ __forceinline__ uint32_t pack_half2_sat(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ void stf(__half* p, float v) {
    unsigned short h;
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(v));
    *reinterpret_cast<unsigned short*>(p) = h;
}
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ld4(const __half* p) {            // 8-byte aligned
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4(__half* p, float4 v) {           // 8-byte aligned
    uint2 u;
    u.x = pack_half2_sat(v.x, v.y);
    u.y = pack_half2_sat(v.z, v.w);
    *reinterpret_cast<uint2*>(p) = u;
}
// value as it will be read back from storage of type T (statistics must see the stored value)
__device__ __forceinline__ float stored(float v, const float*) { return v; }
__device__ __forceinline__ float stored(float v, const __half*) {
    unsigned short h;
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(v));
    return __half2float(__ushort_as_half(h));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// (b, f, t) index of a pixel walking a [B][F][T] grid with a fixed stride: one decomposition up front, then carries only
// (64-bit div/mod per pixel costs ~100 instructions and was the limiter of the HBM-bound elementwise / thin kernels).
struct PixelWalk {
    int t, f, b;          // current position
    int dt, df, db;       // stride decomposed the same way
    int T, F;
    __device__ __forceinline__ void init(int64_t pix, int64_t step, int T_, int F_) {
        T = T_; F = F_;
        t = (int)(pix % T); const int64_t r = pix / T; f = (int)(r % F); b = (int)(r / F);
        dt = (int)(step % T); const int64_t rs = step / T; df = (int)(rs % F); db = (int)(rs / F);
    }
    __device__ __forceinline__ void next() {
        t += dt;
        int cf = 0;
        if (t >= T) { t -= T; cf = 1; }
        f += df + cf;
        int cb = 0;
        if (f >= F) { f -= F; cb = 1; }
        b += db + cb;
    }
};

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

}  // namespace aero
