// Persistent recurrent kernel for one bidirectional LSTM layer (see include/aero_b200.h).
//
// One CTA owns NT sequences (windows) of one direction for all `steps` time steps: W_hh stays
// resident in shared memory (transposed, [j][gate-column]), h lives in shared memory, c in
// registers.  4H threads: thread g accumulates gate column g for the NT sequences
// (acc[n] = sum_j W_hh[g][j] * h[n][j]); the cell update is then spread over the same threads.
// Gate pre-activations from the input projection are prefetched from HBM at the top of each
// step so that their latency hides behind the recurrent mat-vec.
#include "common.cuh"

namespace aero {

template <int H, int NT, typename TO>
__global__ void __launch_bounds__(4 * H) lstm_rec_kernel(const float* __restrict__ gin, const float* __restrict__ bias_pad,
                                                         const float* __restrict__ whh, TO* __restrict__ hout,
                                                         const aero_lstm_params p) {
    constexpr int G = 4 * H;
    constexpr int Q = (NT * H) / G;                    // cell items per thread = NT/4
    static_assert(NT % 4 == 0, "NT must be a multiple of 4");
    extern __shared__ __align__(16) float smem[];
    float* Ws = smem;                                  // [H][G]
    float* hs = Ws + H * G;                            // [H][NT]
    float* gs = hs + H * NT;                           // [NT][G]

    const int g = threadIdx.x;
    const int dir = blockIdx.y;
    const int seq0 = blockIdx.x * NT;
    const int n_seq = p.rows * p.n_win;
    const float* w = whh + (size_t)dir * G * H;
    for (int i = g; i < G * H; i += G) {
        const int gg = i / H, j = i - gg * H;
        Ws[j * G + gg] = w[i];
    }
    for (int i = g; i < H * NT; i += G) hs[i] = 0.f;

    // the cell items of this thread: it = g + q*G -> (n = it / H, j = it % H)
    int item_n[Q], item_j[Q];
    float c_state[Q];
    int64_t in_base[Q], out_base[Q];                   // per-sequence bases
    int seq_row[Q], seq_k[Q];
    bool seq_ok[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        const int it = g + q * G;
        item_n[q] = it / H;
        item_j[q] = it - item_n[q] * H;
        c_state[q] = 0.f;
        const int seq = seq0 + item_n[q];
        seq_ok[q] = seq < n_seq;
        const int s = seq_ok[q] ? seq : 0;
        seq_row[q] = s / p.n_win;
        seq_k[q] = s - seq_row[q] * p.n_win;
        in_base[q] = p.in_windowed ? (int64_t)s * p.steps * 2 * G : (int64_t)seq_row[q] * p.T * 2 * G;
        out_base[q] = p.out_windowed ? (int64_t)s * p.steps * 2 * H : (int64_t)seq_row[q] * p.T * 2 * H;
    }
    const int half = p.win_stride / 2;
    __syncthreads();

    for (int s = 0; s < p.steps; ++s) {
        const int pos = dir ? p.steps - 1 - s : s;
        // ---- prefetch the input-projection gates of this step
        float gi[Q][4];
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const float* src;
            if (p.in_windowed) {
                src = gin + in_base[q] + (int64_t)pos * 2 * G + dir * G;
            } else {
                const int frame = seq_k[q] * p.win_stride + pos;
                src = frame < p.T ? gin + in_base[q] + (int64_t)frame * 2 * G + dir * G : bias_pad + dir * G;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) gi[q][u] = seq_ok[q] ? src[u * H + item_j[q]] : 0.f;
        }
        // ---- recurrent mat-vec: gate column g for NT sequences
        float acc[NT];
#pragma unroll
        for (int n = 0; n < NT; ++n) acc[n] = 0.f;
#pragma unroll 4
        for (int j = 0; j < H; ++j) {
            const float wv = Ws[j * G + g];
#pragma unroll
            for (int n = 0; n < NT; n += 4) {
                const float4 hv = *reinterpret_cast<const float4*>(&hs[j * NT + n]);
                acc[n] = fmaf(wv, hv.x, acc[n]);
                acc[n + 1] = fmaf(wv, hv.y, acc[n + 1]);
                acc[n + 2] = fmaf(wv, hv.z, acc[n + 2]);
                acc[n + 3] = fmaf(wv, hv.w, acc[n + 3]);
            }
        }
#pragma unroll
        for (int n = 0; n < NT; ++n) gs[n * G + g] = acc[n];
        __syncthreads();
        // ---- cell update (PyTorch gate order i, f, g, o)
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const int n = item_n[q], j = item_j[q];
            const float* gr = gs + n * G + j;
            const float ig = sigmoid_f(gr[0] + gi[q][0]);
            const float fg = sigmoid_f(gr[H] + gi[q][1]);
            const float gg = tanhf(gr[2 * H] + gi[q][2]);
            const float og = sigmoid_f(gr[3 * H] + gi[q][3]);
            const float c = fg * c_state[q] + ig * gg;
            c_state[q] = c;
            const float h = og * tanhf(c);
            hs[j * NT + n] = h;
            const float hw = ((p.flags & AERO_TG_ROUND_TF32) && sizeof(TO) == 4) ? round_tf32_rna(h) : h;
            if (seq_ok[q]) {
                if (p.out_windowed) {
                    stf(hout + out_base[q] + (int64_t)pos * 2 * H + dir * H + j, hw);
                } else {
                    const int frame = seq_k[q] * p.win_stride + pos;
                    const int lo = (seq_k[q] == 0) ? 0 : half;
                    const int hi = (seq_k[q] == p.n_win - 1) ? p.steps : p.steps - half;
                    if (pos >= lo && pos < hi && frame < p.T)
                        stf(hout + out_base[q] + (int64_t)frame * 2 * H + dir * H + j, hw);
                }
            }
        }
        __syncthreads();
    }
}

template <int H, int NT>
static int launch_lstm(const float* gin, const float* bias_pad, const float* whh, void* hout, const aero_lstm_params& p,
                       cudaStream_t st) {
    const size_t smem = sizeof(float) * ((size_t)H * 4 * H + (size_t)H * NT + (size_t)NT * 4 * H);
    const int n_seq = p.rows * p.n_win;
    dim3 grid(cdiv(n_seq, NT), 2);
    if (p.flags & AERO_TG_OUT_F16) {
        cudaFuncSetAttribute(lstm_rec_kernel<H, NT, __half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        lstm_rec_kernel<H, NT, __half><<<grid, 4 * H, smem, st>>>(gin, bias_pad, whh, static_cast<__half*>(hout), p);
    } else {
        cudaFuncSetAttribute(lstm_rec_kernel<H, NT, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        lstm_rec_kernel<H, NT, float><<<grid, 4 * H, smem, st>>>(gin, bias_pad, whh, static_cast<float*>(hout), p);
    }
    return check_launch("aero_lstm_rec_fwd");
}

int lstm_tc_launch(const void* gin, const float* bias_pad, const void* whh_r, void* hout, const aero_lstm_params& p,
                   cudaStream_t st);
}  // namespace aero

extern "C" int aero_lstm_rec_fwd(const void* gin_, const float* bias_pad, const void* whh, void* hout,
                                 const aero_lstm_params* p, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(gin_ && whh && hout && p, "aero_lstm_rec_fwd: null argument");
    AERO_REQUIRE(!(p->flags & AERO_TG_A_F16) || p->precision == 1, "aero_lstm_rec_fwd: FP16 gate pre-activations need the wgmma recurrence");
    const float* gin = static_cast<const float*>(gin_);
    AERO_REQUIRE(p->rows >= 1 && p->T >= 1 && p->n_win >= 1 && p->steps >= 1, "aero_lstm_rec_fwd: bad sizes");
    AERO_REQUIRE(p->in_windowed || bias_pad, "aero_lstm_rec_fwd: bias_pad required for un-windowed input");
    AERO_REQUIRE(p->n_win == 1 || (p->win_stride >= 2 && p->win_stride % 2 == 0), "aero_lstm_rec_fwd: win_stride");
    AERO_REQUIRE(p->n_win > 1 || p->steps == p->T || p->in_windowed, "aero_lstm_rec_fwd: single window must span T");
    cudaStream_t st = (cudaStream_t)stream;
    if (p->precision == 1) {
        AERO_REQUIRE(bias_pad, "aero_lstm_rec_fwd: bias_pad required");
        return lstm_tc_launch(gin_, bias_pad, whh, hout, *p, st);
    }
    switch (p->H) {
        case 12: return launch_lstm<12, 16>(gin, bias_pad, (const float*)whh, hout, *p, st);
        case 24: return launch_lstm<24, 16>(gin, bias_pad, (const float*)whh, hout, *p, st);
        case 48: return launch_lstm<48, 16>(gin, bias_pad, (const float*)whh, hout, *p, st);
        case 96: return launch_lstm<96, 16>(gin, bias_pad, (const float*)whh, hout, *p, st);
        default:
            set_error("aero_lstm_rec_fwd: hidden size %d not instantiated (12, 24, 48, 96)", p->H);
            return AERO_ERR_UNSUPPORTED;
    }
}
