// GAN loss terms of the adversarial training step (reference src/solver.py:475-520, src/models/discriminators.py:211-244), read and
// differentiated in place on the discriminators' channels-last / segment storage: the LSGAN and hinge terms on the logits and the
// L1 feature-matching terms against the kept real-clip feature maps.  All terms of one pass go in one call through a device table of
// aero_gan_term descriptors.  See include/aero_b200.h for the contracts and DESIGN.md, "The adversarial step".
#include "common.cuh"

namespace aero {

constexpr int kGanThreads = 256;
constexpr int kGanBwdBlocks = 256;   // blocks per term of the backward (grid-stride over the term's storage)

__device__ __forceinline__ bool gan_term_ok(const aero_gan_term& t) {
    return t.n_seg >= 1 && t.H >= 1 && t.C >= 1 && t.halo >= 0 && t.halo + t.H <= t.seg;
}

// value of the adversarial component at one logit (fp32, as the reference computes it)
__device__ __forceinline__ float gan_adv(int kind, float x) {
    switch (kind) {
        case AERO_GAN_LSGAN_REAL:
        case AERO_GAN_LSGAN_GEN: { const float d = 1.f - x; return d * d; }
        case AERO_GAN_LSGAN_FAKE: return x * x;
        case AERO_GAN_HINGE_REAL:
        case AERO_GAN_HINGE_GEN: return fmaxf(1.f - x, 0.f);
        case AERO_GAN_HINGE_FAKE: return fmaxf(1.f + x, 0.f);
        default: return 0.f;
    }
}

// its derivative (relu' = 0 at the kink, as torch.relu's backward)
__device__ __forceinline__ float gan_adv_grad(int kind, float x) {
    switch (kind) {
        case AERO_GAN_LSGAN_REAL:
        case AERO_GAN_LSGAN_GEN: return -2.f * (1.f - x);
        case AERO_GAN_LSGAN_FAKE: return 2.f * x;
        case AERO_GAN_HINGE_REAL:
        case AERO_GAN_HINGE_GEN: return (1.f - x) > 0.f ? -1.f : 0.f;
        case AERO_GAN_HINGE_FAKE: return (1.f + x) > 0.f ? 1.f : 0.f;
        default: return 0.f;
    }
}

__device__ __forceinline__ float sign_f(float d) { return d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f); }

// fixed-order block sum of two doubles; the result is valid in thread 0
__device__ __forceinline__ void block_sum2(double& a, double& b) {
    __shared__ double red[2][kGanThreads / 32];
    a = warp_sum(a);
    b = warp_sum(b);
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { red[0][w] = a; red[1][w] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        a = b = 0.0;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) { a += red[0][k]; b += red[1][k]; }
    }
}

// grid (AERO_GAN_FWD_BLOCKS, n_terms): block (k, t) sums the owned elements e = k*256 + tid + j*AERO_GAN_FWD_BLOCKS*256 of term t
__global__ void __launch_bounds__(kGanThreads) gan_loss_partial_kernel(const aero_gan_term* __restrict__ terms,
                                                                       double* __restrict__ work) {
    const aero_gan_term t = terms[blockIdx.y];
    double sa = 0.0, sl = 0.0;
    if (!gan_term_ok(t)) {
        sa = sl = __longlong_as_double(0x7ff8000000000000ll);
    } else {
        const int64_t n = (int64_t)t.n_seg * t.H * t.C;
        const int64_t step = (int64_t)gridDim.x * blockDim.x;
        int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
        const bool adv = t.adv != AERO_GAN_NONE && t.adv_scale != 0.0;
        const bool l1 = t.ref != nullptr && t.l1_scale != 0.0;
        if (e < n) {
            PixelWalk pw;                                    // (segment, owned row, channel) of e: b = s, f = h, t = c
            pw.init(e, step, t.C, t.H);
            for (; e < n; e += step, pw.next()) {
                const int64_t a = ((int64_t)pw.b * t.seg + t.halo + pw.f) * t.C + pw.t;
                const float x = t.x[a];
                if (adv) sa += (double)gan_adv(t.adv, x);
                if (l1) sl += (double)fabsf(x - t.ref[a]);
            }
        }
    }
    block_sum2(sa, sl);
    if (threadIdx.x == 0) {
        double* w = work + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * 2;
        w[0] = sa;
        w[1] = sl;
    }
}

// one block per term: the AERO_GAN_FWD_BLOCKS partials in a fixed order, scaled
__global__ void __launch_bounds__(AERO_GAN_FWD_BLOCKS) gan_loss_final_kernel(const aero_gan_term* __restrict__ terms,
                                                                             const double* __restrict__ work, double* __restrict__ out) {
    const double* w = work + ((int64_t)blockIdx.x * AERO_GAN_FWD_BLOCKS + threadIdx.x) * 2;
    double sa = w[0], sl = w[1];
    block_sum2(sa, sl);
    if (threadIdx.x == 0) {
        const aero_gan_term& t = terms[blockIdx.x];
        out[2 * blockIdx.x] = t.adv == AERO_GAN_NONE ? sa * 0.0 : t.adv_scale * sa;   // sa * 0: NaN of a bad geometry survives
        out[2 * blockIdx.x + 1] = t.ref == nullptr ? sl * 0.0 : t.l1_scale * sl;
    }
}

// grid (kGanBwdBlocks, n_terms): every element of the term's storage [n_seg][seg][C] written
__global__ void __launch_bounds__(kGanThreads) gan_loss_bwd_kernel(const aero_gan_term* __restrict__ terms) {
    const aero_gan_term t = terms[blockIdx.y];
    if (t.dx == nullptr || t.n_seg < 1 || t.seg < 1 || t.C < 1) return;
    const bool ok = gan_term_ok(t);
    const int kind = t.adv;
    const float sa = (float)t.adv_scale, sl = t.ref != nullptr ? (float)t.l1_scale : 0.f;
    const int64_t n = (int64_t)t.n_seg * t.seg * t.C;
    const int64_t step = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    PixelWalk pw;                                            // b = segment, f = row of the segment, t = channel
    pw.init(i, step, t.C, t.seg);
    for (; i < n; i += step, pw.next()) {
        float g = 0.f;
        const int h = pw.f - t.halo;
        if (!ok) {
            g = __int_as_float(0x7fc00000);
        } else if (h >= 0 && h < t.H) {
            const float x = t.x[i];
            if (kind != AERO_GAN_NONE) g = sa * gan_adv_grad(kind, x);
            if (sl != 0.f) g += sl * sign_f(x - t.ref[i]);
        }
        t.dx[i] = g;
    }
}

}  // namespace aero

extern "C" int aero_gan_loss_fwd(const aero_gan_term* terms, int32_t n_terms, double* out, double* work, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(terms && out && work, "aero_gan_loss_fwd: null argument");
    AERO_REQUIRE(n_terms >= 1 && n_terms <= 65535, "aero_gan_loss_fwd: n_terms=%d", n_terms);
    gan_loss_partial_kernel<<<dim3(AERO_GAN_FWD_BLOCKS, n_terms), kGanThreads, 0, (cudaStream_t)stream>>>(terms, work);
    int rc = check_launch("aero_gan_loss_fwd (partial sums)");
    if (rc != AERO_OK) return rc;
    gan_loss_final_kernel<<<n_terms, AERO_GAN_FWD_BLOCKS, 0, (cudaStream_t)stream>>>(terms, work, out);
    return check_launch("aero_gan_loss_fwd");
}

extern "C" int aero_gan_loss_bwd(const aero_gan_term* terms, int32_t n_terms, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(terms, "aero_gan_loss_bwd: null argument");
    AERO_REQUIRE(n_terms >= 1 && n_terms <= 65535, "aero_gan_loss_bwd: n_terms=%d", n_terms);
    gan_loss_bwd_kernel<<<dim3(kGanBwdBlocks, n_terms), kGanThreads, 0, (cudaStream_t)stream>>>(terms);
    return check_launch("aero_gan_loss_bwd");
}
