// LocalState attention core on the warp-level tensor path (mma.sync m16n8k8 TF32, fp32 accumulate), FA2-style.
// Used when aero_attn_params.flags has AERO_TG_ROUND_TF32 (the engine's tensor-core mode); attention.cu is the exact-fp32 twin.
//
// One CTA = one (row, head) and 64 queries (4 warps x 16).  K and V of that (row, head) stream through shared memory in
// double-buffered tiles of 64 keys filled by cp.async (16-byte chunks, zero fill past T) while the previous tile is being
// consumed; the producing GEMM rounds q/k/v to TF32, so no conversion is needed on the way.  Per block of 8 keys a warp issues
//   S[16 q x 8 keys]  = Q[16 x d] K^T        (d/8 mma, Q fragments live in registers, pre-scaled by log2(e)/sqrt(d))
//   O[16 q x d]      += P[16 x 8] V[8 x d]   (d/8 mma)
// The C-fragment of S is reused directly as the A-fragment of P by permuting the key order inside the block
// (k = tig <-> key 2 tig, k = tig + 4 <-> key 2 tig + 1), so no shuffles are needed between the two products.
// Scores live in the log2 domain: s = q.k * log2e/sqrt(d) - |t - s| * slope * log2e, diagonal = -100 * log2e, p = 2^(s - m).
// Online softmax over chunks of 32 keys (one max reduction + one accumulator rescale per chunk).
#include "common.cuh"

namespace aero {

constexpr int kAQ = 64;      // queries per CTA
constexpr int kAKT = 64;     // keys per smem tile (two buffers)
constexpr float kLog2e = 1.4426950408889634f;

// round-to-nearest TF32 bit pattern in two integer instructions (ptxas expands cvt.rna.tf32.f32 into ~5)
__device__ __forceinline__ uint32_t to_tf32(float x) { return (__float_as_uint(x) + 0x1000u) & 0xffffe000u; }
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float ex2f(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Rows are p.T frames apart; the first Tr of them take part (Tr = p.T, or the row's own length in a ragged batch).
template <int D, typename TO>   // head dim: 12 or 24
__device__ __forceinline__ void local_attn_mma_block(const float* __restrict__ qkvd, TO* __restrict__ out,
                                                     const aero_attn_params& p, const int Tr) {
    constexpr int DP = (D + 7) / 8 * 8;                  // 16 or 24
    constexpr int KS = DP / 8;                           // k-steps of QK^T == n-tiles of PV
    constexpr int PITCH = DP + 4;                        // 20 / 28: conflict-free fragment loads
    __shared__ __align__(16) uint32_t Ksm[2][kAKT * PITCH];
    __shared__ __align__(16) uint32_t Vsm[2][kAKT * PITCH];
    constexpr int CH = D / 4;                            // 16-byte chunks per key row (D = 12 / 24)
    for (int i = threadIdx.x; i < 2 * kAKT * PITCH; i += 128) { (&Ksm[0][0])[i] = 0u; (&Vsm[0][0])[i] = 0u; }   // padding columns stay zero
    __syncthreads();

    const int row = blockIdx.z, h = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, tig = lane & 3;
    const int q0 = blockIdx.x * kAQ + warp * 16;         // first query of this warp
    const float* base = qkvd + (int64_t)row * p.T * p.ld;

    // ---- Q fragments (A operand), rows g / g+8, pre-scaled so that scores come out in the log2 domain
    const int s_lo = q0 + g, s_hi = q0 + g + 8;
    const int sl = min(s_lo, Tr - 1), sh = min(s_hi, Tr - 1);
    const float qs = kLog2e * rsqrtf((float)D);
    uint32_t qa[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
        const int d0 = ks * 8 + tig, d1 = d0 + 4;
        qa[ks][0] = to_tf32(d0 < D ? base[(int64_t)sl * p.ld + h * D + d0] * qs : 0.f);
        qa[ks][1] = to_tf32(d0 < D ? base[(int64_t)sh * p.ld + h * D + d0] * qs : 0.f);
        qa[ks][2] = to_tf32(d1 < D ? base[(int64_t)sl * p.ld + h * D + d1] * qs : 0.f);
        qa[ks][3] = to_tf32(d1 < D ? base[(int64_t)sh * p.ld + h * D + d1] * qs : 0.f);
    }
    // decay slope per query (reference modules.py:111-117), in the log2 domain
    float slope_lo = 0.f, slope_hi = 0.f;
    for (int f = 0; f < p.ndecay; ++f) {
        slope_lo += (float)(f + 1) * 0.5f * sigmoid_f(base[(int64_t)sl * p.ld + 3 * p.H + h * p.ndecay + f]);
        slope_hi += (float)(f + 1) * 0.5f * sigmoid_f(base[(int64_t)sh * p.ld + 3 * p.H + h * p.ndecay + f]);
    }
    const float rs = rsqrtf((float)p.ndecay) * kLog2e;
    slope_lo *= rs;
    slope_hi *= rs;

    float o[KS][4];
#pragma unroll
    for (int nt = 0; nt < KS; ++nt) { o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f; }
    float m_lo = -1e30f, m_hi = -1e30f, l_lo = 0.f, l_hi = 0.f;
    constexpr float kDiag = -100.0f * kLog2e;

    // asynchronous fill of one tile: key rows beyond T are zero-filled (src-size 0)
    auto fill = [&](int k0, int buf) {
        for (int i = threadIdx.x; i < kAKT * CH * 2; i += 128) {
            const int which = i / (kAKT * CH), j = i - which * (kAKT * CH);
            const int t = j / CH, c4 = j - t * CH;
            const bool ok = k0 + t < Tr;
            const float* src = base + (int64_t)min(k0 + t, Tr - 1) * p.ld + (which + 1) * p.H + h * D + 4 * c4;
            const uint32_t dst = (uint32_t)__cvta_generic_to_shared((which ? &Vsm[buf][0] : &Ksm[buf][0]) + t * PITCH + 4 * c4);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    fill(0, 0);
    int it = 0;
    for (int k0 = 0; k0 < Tr; k0 += kAKT, ++it) {
        const int nk = min(kAKT, Tr - k0);
        if (k0 + kAKT < Tr) fill(k0 + kAKT, (it + 1) & 1);
        else asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncthreads();
        const uint32_t* Ks = &Ksm[it & 1][0];
        const uint32_t* Vs = &Vsm[it & 1][0];
        const int nblk = (nk + 7) >> 3;
        for (int cb = 0; cb < nblk; cb += 4) {               // chunk of up to 4 key blocks = 32 keys
            float sc[4][4];
            float cm_lo = -1e30f, cm_hi = -1e30f;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int kb = cb + u;
                sc[u][0] = sc[u][1] = sc[u][2] = sc[u][3] = 0.f;
                if (kb < nblk) {
#pragma unroll
                    for (int ks = 0; ks < KS; ++ks) {
                        const uint32_t b0 = Ks[(kb * 8 + g) * PITCH + ks * 8 + tig];
                        const uint32_t b1 = Ks[(kb * 8 + g) * PITCH + ks * 8 + tig + 4];
                        mma_tf32(sc[u], qa[ks], b0, b1);
                    }
                    // c0: (row g, key 2 tig)  c1: (row g, key 2 tig + 1)  c2, c3: row g + 8
                    const int t_a = k0 + kb * 8 + 2 * tig;
                    const float d_lo = (float)(t_a - s_lo), d_hi = (float)(t_a - s_hi);
                    sc[u][0] = fmaf(-fabsf(d_lo), slope_lo, sc[u][0]);
                    sc[u][1] = fmaf(-fabsf(d_lo + 1.f), slope_lo, sc[u][1]);
                    sc[u][2] = fmaf(-fabsf(d_hi), slope_hi, sc[u][2]);
                    sc[u][3] = fmaf(-fabsf(d_hi + 1.f), slope_hi, sc[u][3]);
                    // the diagonal and the padding keys touch one or two key blocks per warp: keep them off the common path
                    const int kb0 = k0 + kb * 8;                                       // (warp-uniform)
                    if (kb0 < q0 + 16 && kb0 + 8 > q0) {
                        if (t_a == s_lo) sc[u][0] = kDiag;
                        if (t_a + 1 == s_lo) sc[u][1] = kDiag;
                        if (t_a == s_hi) sc[u][2] = kDiag;
                        if (t_a + 1 == s_hi) sc[u][3] = kDiag;
                    }
                    if (kb0 + 8 > Tr) {                                               // padding keys of the last block
                        if (t_a >= Tr) { sc[u][0] = -1e30f; sc[u][2] = -1e30f; }
                        if (t_a + 1 >= Tr) { sc[u][1] = -1e30f; sc[u][3] = -1e30f; }
                    }
                    cm_lo = fmaxf(cm_lo, fmaxf(sc[u][0], sc[u][1]));
                    cm_hi = fmaxf(cm_hi, fmaxf(sc[u][2], sc[u][3]));
                } else {
                    sc[u][0] = sc[u][1] = sc[u][2] = sc[u][3] = -1e30f;
                }
            }
            // row maxima across the 4 lanes of a quad, then one rescale per chunk
            cm_lo = fmaxf(cm_lo, __shfl_xor_sync(0xffffffffu, cm_lo, 1));
            cm_lo = fmaxf(cm_lo, __shfl_xor_sync(0xffffffffu, cm_lo, 2));
            cm_hi = fmaxf(cm_hi, __shfl_xor_sync(0xffffffffu, cm_hi, 1));
            cm_hi = fmaxf(cm_hi, __shfl_xor_sync(0xffffffffu, cm_hi, 2));
            const float mn_lo = fmaxf(m_lo, cm_lo), mn_hi = fmaxf(m_hi, cm_hi);
            const float cr_lo = ex2f(m_lo - mn_lo), cr_hi = ex2f(m_hi - mn_hi);
            m_lo = mn_lo; m_hi = mn_hi;
            l_lo *= cr_lo; l_hi *= cr_hi;
#pragma unroll
            for (int nt = 0; nt < KS; ++nt) { o[nt][0] *= cr_lo; o[nt][1] *= cr_lo; o[nt][2] *= cr_hi; o[nt][3] *= cr_hi; }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int kb = cb + u;
                if (kb >= nblk) break;
                const float p0 = ex2f(sc[u][0] - m_lo), p1 = ex2f(sc[u][1] - m_lo);
                const float p2 = ex2f(sc[u][2] - m_hi), p3 = ex2f(sc[u][3] - m_hi);
                l_lo += p0 + p1;
                l_hi += p2 + p3;
                // A fragment of P with the permuted key order: (g, k=tig) = key 2tig, (g+8, k=tig), (g, k=tig+4) = key 2tig+1, (g+8, ..)
                const uint32_t pa[4] = {to_tf32(p0), to_tf32(p2), to_tf32(p1), to_tf32(p3)};
#pragma unroll
                for (int nt = 0; nt < KS; ++nt) {
                    const uint32_t b0 = Vs[(kb * 8 + 2 * tig) * PITCH + nt * 8 + g];
                    const uint32_t b1 = Vs[(kb * 8 + 2 * tig + 1) * PITCH + nt * 8 + g];
                    mma_tf32(o[nt], pa, b0, b1);
                }
            }
        }
        __syncthreads();                                 // this buffer is refilled by the prefetch issued one iteration from now
    }
    // row sums across the quad, normalise, store (C fragment: cols nt*8 + 2 tig, +1)
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1); l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1); l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float il_lo = 1.0f / l_lo, il_hi = 1.0f / l_hi;
#pragma unroll
    for (int nt = 0; nt < KS; ++nt) {
        const int c = nt * 8 + 2 * tig;
        if (c < D) {
            if (s_lo < Tr) {
                TO* op = out + ((int64_t)row * p.T + s_lo) * p.H + h * D + c;
                stf(op, round_tf32_rna(o[nt][0] * il_lo));
                if (c + 1 < D) stf(op + 1, round_tf32_rna(o[nt][1] * il_lo));
            }
            if (s_hi < Tr) {
                TO* op = out + ((int64_t)row * p.T + s_hi) * p.H + h * D + c;
                stf(op, round_tf32_rna(o[nt][2] * il_hi));
                if (c + 1 < D) stf(op + 1, round_tf32_rna(o[nt][3] * il_hi));
            }
        }
    }
}

template <int D, typename TO>
__global__ void __launch_bounds__(128) local_attn_mma_kernel(const float* __restrict__ qkvd, TO* __restrict__ out,
                                                             const aero_attn_params p) {
    local_attn_mma_block<D, TO>(qkvd, out, p, p.T);
}

// ragged batch: row r belongs to clip r / rows_per_clip, whose first frames[clip] frames are valid
template <int D, typename TO>
__global__ void __launch_bounds__(128) local_attn_mma_varlen_kernel(const float* __restrict__ qkvd, TO* __restrict__ out,
                                                                    const int32_t* __restrict__ frames, const int rows_per_clip,
                                                                    const aero_attn_params p) {
    const int Tr = frames[blockIdx.z / rows_per_clip];
    if ((int)blockIdx.x * kAQ >= Tr) return;
    local_attn_mma_block<D, TO>(qkvd, out, p, Tr);
}

// frames != nullptr: ragged batch (aero_local_attn_varlen_fwd)
int local_attn_mma_launch(const float* qkvd, void* out, const aero_attn_params& p, cudaStream_t st, bool* taken,
                          const int32_t* frames, int rows_per_clip) {
    const int d = p.H / p.heads;
    *taken = (d == 12 || d == 24) && p.ld % 4 == 0 && p.H % 4 == 0 && (reinterpret_cast<uintptr_t>(qkvd) & 15) == 0;   // 16-byte cp.async chunks
    if (!*taken) return AERO_OK;
    dim3 grid(cdiv(p.T, kAQ), p.heads, p.rows);
    if (frames) {
        if (p.flags & AERO_TG_OUT_F16) {
            if (d == 12) local_attn_mma_varlen_kernel<12, __half><<<grid, 128, 0, st>>>(qkvd, static_cast<__half*>(out), frames, rows_per_clip, p);
            else local_attn_mma_varlen_kernel<24, __half><<<grid, 128, 0, st>>>(qkvd, static_cast<__half*>(out), frames, rows_per_clip, p);
        } else {
            if (d == 12) local_attn_mma_varlen_kernel<12, float><<<grid, 128, 0, st>>>(qkvd, static_cast<float*>(out), frames, rows_per_clip, p);
            else local_attn_mma_varlen_kernel<24, float><<<grid, 128, 0, st>>>(qkvd, static_cast<float*>(out), frames, rows_per_clip, p);
        }
        return check_launch("aero_local_attn_varlen_fwd(mma)");
    }
    if (p.flags & AERO_TG_OUT_F16) {
        if (d == 12) local_attn_mma_kernel<12, __half><<<grid, 128, 0, st>>>(qkvd, static_cast<__half*>(out), p);
        else local_attn_mma_kernel<24, __half><<<grid, 128, 0, st>>>(qkvd, static_cast<__half*>(out), p);
    } else {
        if (d == 12) local_attn_mma_kernel<12, float><<<grid, 128, 0, st>>>(qkvd, static_cast<float*>(out), p);
        else local_attn_mma_kernel<24, float><<<grid, 128, 0, st>>>(qkvd, static_cast<float*>(out), p);
    }
    return check_launch("aero_local_attn_fwd(mma)");
}

}  // namespace aero
