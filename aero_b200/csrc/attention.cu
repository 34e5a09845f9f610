// LocalState attention core (see include/aero_b200.h): flash-style, one thread per query, keys and
// values streamed through shared memory in tiles, online softmax over the key axis, the decay
// penalty -|t-s|*slope[s] and the -100 diagonal applied on the fly.  No T x T tensor in HBM.
#include "common.cuh"

namespace aero {

constexpr int kQB = 128;     // queries per CTA (one per thread)
constexpr int kKT = 256;     // keys per shared-memory tile

// Rows are p.T frames apart; the first Tr of them take part (Tr = p.T, or the row's own length in a ragged batch).
template <int D, typename TO>
__device__ __forceinline__ void local_attn_block(const float* __restrict__ qkvd, TO* __restrict__ out,
                                                 const aero_attn_params& p, const int Tr) {
    __shared__ __align__(16) float Ks[kKT * D];
    __shared__ __align__(16) float Vs[kKT * D];
    const int row = blockIdx.z, h = blockIdx.y;
    const int s = blockIdx.x * kQB + threadIdx.x;
    const bool valid = s < Tr;
    const int sq = valid ? s : Tr - 1;
    const float* base = qkvd + (int64_t)row * p.T * p.ld;

    float q[D];
    const float inv = rsqrtf((float)D);
#pragma unroll
    for (int c = 0; c < D; ++c) q[c] = base[(int64_t)sq * p.ld + h * D + c] * inv;
    float slope = 0.f;
    for (int f = 0; f < p.ndecay; ++f)
        slope += (float)(f + 1) * 0.5f * sigmoid_f(base[(int64_t)sq * p.ld + 3 * p.H + h * p.ndecay + f]);
    slope *= rsqrtf((float)p.ndecay);

    float m = -1e30f, l = 0.f, acc[D];
#pragma unroll
    for (int c = 0; c < D; ++c) acc[c] = 0.f;

    for (int k0 = 0; k0 < Tr; k0 += kKT) {
        const int nk = min(kKT, Tr - k0);
        __syncthreads();
        for (int i = threadIdx.x; i < nk * D; i += kQB) {
            const int t = i / D, c = i - t * D;
            const float* src = base + (int64_t)(k0 + t) * p.ld + h * D + c;
            Ks[i] = src[p.H];
            Vs[i] = src[2 * p.H];
        }
        __syncthreads();
        for (int t0 = 0; t0 < nk; t0 += 8) {
            float sc[8];
            float cm = -1e30f;
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int t = t0 + u;
                float d = -1e30f;
                if (t < nk) {
                    d = 0.f;
#pragma unroll
                    for (int c = 0; c < D; ++c) d = fmaf(q[c], Ks[t * D + c], d);
                    const int ta = k0 + t;
                    d -= fabsf((float)(ta - sq)) * slope;
                    if (ta == sq) d = -100.0f;
                }
                sc[u] = d;
                cm = fmaxf(cm, d);
            }
            const float mn = fmaxf(m, cm);
            const float corr = __expf(m - mn);
            l *= corr;
#pragma unroll
            for (int c = 0; c < D; ++c) acc[c] *= corr;
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int t = t0 + u;
                if (t < nk) {
                    const float pr = __expf(sc[u] - mn);
                    l += pr;
#pragma unroll
                    for (int c = 0; c < D; ++c) acc[c] = fmaf(pr, Vs[t * D + c], acc[c]);
                }
            }
            m = mn;
        }
    }
    if (valid) {
        const float il = 1.0f / l;
        TO* o = out + ((int64_t)row * p.T + s) * p.H + h * D;
        const bool rnd = (p.flags & AERO_TG_ROUND_TF32) && sizeof(TO) == 4;
#pragma unroll
        for (int c = 0; c < D; ++c) stf(o + c, rnd ? round_tf32_rna(acc[c] * il) : acc[c] * il);
    }
}

template <int D, typename TO>
__global__ void __launch_bounds__(kQB) local_attn_kernel(const float* __restrict__ qkvd, TO* __restrict__ out,
                                                         const aero_attn_params p) {
    local_attn_block<D, TO>(qkvd, out, p, p.T);
}

// ragged batch: row r belongs to clip r / rows_per_clip, whose first frames[clip] frames are valid
template <int D, typename TO>
__global__ void __launch_bounds__(kQB) local_attn_varlen_kernel(const float* __restrict__ qkvd, TO* __restrict__ out,
                                                                const int32_t* __restrict__ frames, const int rows_per_clip,
                                                                const aero_attn_params p) {
    const int Tr = frames[blockIdx.z / rows_per_clip];
    if ((int)blockIdx.x * kQB >= Tr) return;
    local_attn_block<D, TO>(qkvd, out, p, Tr);
}

template <int D>
static int launch_attn(const float* qkvd, void* out, const aero_attn_params& p, cudaStream_t st) {
    dim3 grid(cdiv(p.T, kQB), p.heads, p.rows);
    if (p.flags & AERO_TG_OUT_F16) local_attn_kernel<D, __half><<<grid, kQB, 0, st>>>(qkvd, static_cast<__half*>(out), p);
    else local_attn_kernel<D, float><<<grid, kQB, 0, st>>>(qkvd, static_cast<float*>(out), p);
    return check_launch("aero_local_attn_fwd");
}

template <int D>
static int launch_attn_varlen(const float* qkvd, void* out, const int32_t* frames, int rows_per_clip, const aero_attn_params& p,
                              cudaStream_t st) {
    dim3 grid(cdiv(p.T, kQB), p.heads, p.rows);
    if (p.flags & AERO_TG_OUT_F16)
        local_attn_varlen_kernel<D, __half><<<grid, kQB, 0, st>>>(qkvd, static_cast<__half*>(out), frames, rows_per_clip, p);
    else
        local_attn_varlen_kernel<D, float><<<grid, kQB, 0, st>>>(qkvd, static_cast<float*>(out), frames, rows_per_clip, p);
    return check_launch("aero_local_attn_varlen_fwd");
}

int local_attn_mma_launch(const float* qkvd, void* out, const aero_attn_params& p, cudaStream_t st, bool* taken,
                          const int32_t* frames, int rows_per_clip);
}  // namespace aero

extern "C" int aero_local_attn_fwd(const float* qkvd, void* out, const aero_attn_params* p, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(qkvd && out && p, "aero_local_attn_fwd: null argument");
    AERO_REQUIRE(p->heads >= 1 && p->H % p->heads == 0 && p->ndecay >= 1 && p->ndecay <= 16, "aero_local_attn_fwd: heads/ndecay");
    AERO_REQUIRE(p->ld >= 3 * p->H + p->heads * p->ndecay, "aero_local_attn_fwd: ld=%d too small", p->ld);
    AERO_REQUIRE(p->rows >= 1 && p->rows <= 65535 && p->T >= 1, "aero_local_attn_fwd: rows=%d", p->rows);
    cudaStream_t st = (cudaStream_t)stream;
    if (p->flags & AERO_TG_ROUND_TF32) {            // tensor-core mode: TF32 mma.sync kernel (attention_mma.cu)
        bool taken = false;
        const int rc = local_attn_mma_launch(qkvd, out, *p, st, &taken, nullptr, 0);
        if (taken || rc != AERO_OK) return rc;
    }
    switch (p->H / p->heads) {
        case 3: return launch_attn<3>(qkvd, out, *p, st);
        case 6: return launch_attn<6>(qkvd, out, *p, st);
        case 12: return launch_attn<12>(qkvd, out, *p, st);
        case 24: return launch_attn<24>(qkvd, out, *p, st);
        default:
            set_error("aero_local_attn_fwd: head dim %d not instantiated (3, 6, 12, 24)", p->H / p->heads);
            return AERO_ERR_UNSUPPORTED;
    }
}

extern "C" int aero_local_attn_varlen_fwd(const float* qkvd, void* out, const int32_t* frames, int32_t rows_per_clip,
                                          const aero_attn_params* p, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(qkvd && out && frames && p, "aero_local_attn_varlen_fwd: null argument");
    AERO_REQUIRE(p->heads >= 1 && p->H % p->heads == 0 && p->ndecay >= 1 && p->ndecay <= 16, "aero_local_attn_varlen_fwd: heads/ndecay");
    AERO_REQUIRE(p->ld >= 3 * p->H + p->heads * p->ndecay, "aero_local_attn_varlen_fwd: ld=%d too small", p->ld);
    AERO_REQUIRE(p->rows >= 1 && p->rows <= 65535 && p->T >= 1, "aero_local_attn_varlen_fwd: rows=%d", p->rows);
    AERO_REQUIRE(rows_per_clip >= 1 && p->rows % rows_per_clip == 0, "aero_local_attn_varlen_fwd: rows_per_clip=%d", rows_per_clip);
    cudaStream_t st = (cudaStream_t)stream;
    if (p->flags & AERO_TG_ROUND_TF32) {
        bool taken = false;
        const int rc = local_attn_mma_launch(qkvd, out, *p, st, &taken, frames, rows_per_clip);
        if (taken || rc != AERO_OK) return rc;
    }
    switch (p->H / p->heads) {
        case 3: return launch_attn_varlen<3>(qkvd, out, frames, rows_per_clip, *p, st);
        case 6: return launch_attn_varlen<6>(qkvd, out, frames, rows_per_clip, *p, st);
        case 12: return launch_attn_varlen<12>(qkvd, out, frames, rows_per_clip, *p, st);
        case 24: return launch_attn_varlen<24>(qkvd, out, frames, rows_per_clip, *p, st);
        default:
            set_error("aero_local_attn_varlen_fwd: head dim %d not instantiated (3, 6, 12, 24)", p->H / p->heads);
            return AERO_ERR_UNSUPPORTED;
    }
}
