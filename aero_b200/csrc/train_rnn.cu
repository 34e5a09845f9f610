// Training form of the bidirectional LSTM layer (reference modules.py:28-65 under autograd; replaces cuDNN's RNN forward-
// for-training and backward-data kernels).  fp32, one CTA per NT sequences (windows) of one direction, W_hh resident in
// shared memory, like the inference SIMT recurrence (lstm.cu).
//   forward : as aero_lstm_rec_fwd (precision 0), and additionally saves, in the WINDOWED layout [n_seq][steps][2][..],
//             the post-activation gates (i, f, g, o), the cell state c and the hidden state h of every step.
//   backward: back-propagation through time.  Per step: d(gates) from the saved activations, written windowed as
//             dgin[n_seq][steps][2][4H] (the gradient of the gate pre-activations, i.e. of the input projection's output),
//             then dh_{t-1} = d(gates) . W_hh as a small shared-memory mat-vec.  Weight / bias / input gradients are
//             GEMMs over dgin done by the caller (aero_tapgemm_wgrad / aero_colsum / aero_tapgemm_fwd).
//   fold    : sums the windowed dgin over the overlapping windows back onto the un-windowed frames (first layer).
#include "common.cuh"

namespace aero {

template <int H, int NT>
__global__ void __launch_bounds__(4 * H) lstm_train_fwd_kernel(const float* __restrict__ gin, const float* __restrict__ bias_pad,
                                                               const float* __restrict__ whh, float* __restrict__ hout,
                                                               float* __restrict__ gates_s, float* __restrict__ c_s,
                                                               float* __restrict__ h_s, const aero_lstm_params p) {
    constexpr int G = 4 * H;
    constexpr int Q = (NT * H) / G;
    extern __shared__ __align__(16) float smem[];
    float* Ws = smem;                                  // [H][G]  (transposed: Ws[j*G + g])
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
    int item_n[Q], item_j[Q], seq_row[Q], seq_k[Q], seq_id[Q];
    float c_state[Q];
    bool seq_ok[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        const int it = g + q * G;
        item_n[q] = it / H;
        item_j[q] = it - item_n[q] * H;
        c_state[q] = 0.f;
        const int seq = seq0 + item_n[q];
        seq_ok[q] = seq < n_seq;
        seq_id[q] = seq_ok[q] ? seq : 0;
        seq_row[q] = seq_id[q] / p.n_win;
        seq_k[q] = seq_id[q] - seq_row[q] * p.n_win;
    }
    const int half = p.win_stride / 2;
    __syncthreads();
    for (int s = 0; s < p.steps; ++s) {
        const int pos = dir ? p.steps - 1 - s : s;
        float gi[Q][4];
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const float* src;
            if (p.in_windowed) {
                src = gin + ((int64_t)seq_id[q] * p.steps + pos) * 2 * G + dir * G;
            } else {
                const int frame = seq_k[q] * p.win_stride + pos;
                src = frame < p.T ? gin + ((int64_t)seq_row[q] * p.T + frame) * 2 * G + dir * G : bias_pad + dir * G;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) gi[q][u] = seq_ok[q] ? src[u * H + item_j[q]] : 0.f;
        }
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
            if (seq_ok[q]) {
                const int64_t wpos = ((int64_t)seq_id[q] * p.steps + pos) * 2 + dir;
                float* gd = gates_s + wpos * G + j;
                gd[0] = ig; gd[H] = fg; gd[2 * H] = gg; gd[3 * H] = og;
                c_s[wpos * H + j] = c;
                h_s[wpos * H + j] = h;
                if (hout && !p.out_windowed) {
                    const int frame = seq_k[q] * p.win_stride + pos;
                    const int lo = (seq_k[q] == 0) ? 0 : half;
                    const int hi = (seq_k[q] == p.n_win - 1) ? p.steps : p.steps - half;
                    if (pos >= lo && pos < hi && frame < p.T) hout[((int64_t)seq_row[q] * p.T + frame) * 2 * H + dir * H + j] = h;
                }
            }
        }
        __syncthreads();
    }
}

template <int H, int NT>
__global__ void __launch_bounds__(4 * H) lstm_bwd_kernel(const float* __restrict__ dhout, const float* __restrict__ gates_s,
                                                         const float* __restrict__ c_s, const float* __restrict__ whh,
                                                         float* __restrict__ dgin_w, const aero_lstm_params p) {
    constexpr int G = 4 * H;
    constexpr int Q = (NT * H) / G;
    extern __shared__ __align__(16) float smem[];
    float* Ws = smem;                                  // [G][H] (as stored: Ws[g*H + j])
    float* dgs = Ws + G * H;                           // [NT][G]
    float* dhr = dgs + NT * G;                         // [NT][H]
    const int tid = threadIdx.x;
    const int dir = blockIdx.y;
    const int seq0 = blockIdx.x * NT;
    const int n_seq = p.rows * p.n_win;
    const float* w = whh + (size_t)dir * G * H;
    for (int i = tid; i < G * H; i += G) Ws[i] = w[i];
    for (int i = tid; i < NT * H; i += G) dhr[i] = 0.f;
    int item_n[Q], item_j[Q], seq_row[Q], seq_k[Q], seq_id[Q];
    float dc_state[Q];
    bool seq_ok[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        const int it = tid + q * G;
        item_n[q] = it / H;
        item_j[q] = it - item_n[q] * H;
        dc_state[q] = 0.f;
        const int seq = seq0 + item_n[q];
        seq_ok[q] = seq < n_seq;
        seq_id[q] = seq_ok[q] ? seq : 0;
        seq_row[q] = seq_id[q] / p.n_win;
        seq_k[q] = seq_id[q] - seq_row[q] * p.n_win;
    }
    const int half = p.win_stride / 2;
    // inputs of one step of one cell item; loaded one step ahead so that the HBM / L2 latency hides behind the mat-vec
    struct StepIn { float ig, fg, gg, og, c, c_prev, dh_ext; };
    auto load_step = [&](int s, int q) -> StepIn {
        StepIn v = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (s < 0 || !seq_ok[q]) return v;
        const int pos = dir ? p.steps - 1 - s : s;
        const int pos_prev = dir ? pos + 1 : pos - 1;              // position processed one step earlier (s - 1)
        const int j = item_j[q];
        if (p.out_windowed) {
            v.dh_ext = dhout[((int64_t)seq_id[q] * p.steps + pos) * 2 * H + dir * H + j];
        } else {
            const int frame = seq_k[q] * p.win_stride + pos;
            const int lo = (seq_k[q] == 0) ? 0 : half;
            const int hi = (seq_k[q] == p.n_win - 1) ? p.steps : p.steps - half;
            if (pos >= lo && pos < hi && frame < p.T) v.dh_ext = dhout[((int64_t)seq_row[q] * p.T + frame) * 2 * H + dir * H + j];
        }
        const int64_t wpos = ((int64_t)seq_id[q] * p.steps + pos) * 2 + dir;
        const float* gd = gates_s + wpos * G + j;
        v.ig = gd[0]; v.fg = gd[H]; v.gg = gd[2 * H]; v.og = gd[3 * H];
        v.c = c_s[wpos * H + j];
        v.c_prev = (s > 0) ? c_s[(((int64_t)seq_id[q] * p.steps + pos_prev) * 2 + dir) * H + j] : 0.f;
        return v;
    };
    StepIn cur[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) cur[q] = load_step(p.steps - 1, q);
    __syncthreads();
    for (int s = p.steps - 1; s >= 0; --s) {
        const int pos = dir ? p.steps - 1 - s : s;
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const int n = item_n[q], j = item_j[q];
            float d_ig = 0.f, d_fg = 0.f, d_gg = 0.f, d_og = 0.f;
            if (seq_ok[q]) {
                const float dh = dhr[n * H + j] + cur[q].dh_ext;
                const float ig = cur[q].ig, fg = cur[q].fg, gg = cur[q].gg, og = cur[q].og;
                const float th = tanhf(cur[q].c);
                const float dc = dh * og * (1.0f - th * th) + dc_state[q];
                d_og = dh * th * og * (1.0f - og);
                d_ig = dc * gg * ig * (1.0f - ig);
                d_fg = dc * cur[q].c_prev * fg * (1.0f - fg);
                d_gg = dc * ig * (1.0f - gg * gg);
                dc_state[q] = dc * fg;
                const int64_t wpos = ((int64_t)seq_id[q] * p.steps + pos) * 2 + dir;
                float* dd = dgin_w + wpos * G + j;
                dd[0] = d_ig; dd[H] = d_fg; dd[2 * H] = d_gg; dd[3 * H] = d_og;
            }
            float* ds = dgs + n * G + j;
            ds[0] = d_ig; ds[H] = d_fg; ds[2 * H] = d_gg; ds[3 * H] = d_og;
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < Q; ++q) cur[q] = load_step(s - 1, q);          // issued now, consumed after the mat-vec
        if (s > 0) {
            float acc[Q];
#pragma unroll
            for (int q = 0; q < Q; ++q) acc[q] = 0.f;
#pragma unroll 4
            for (int gg = 0; gg < G; ++gg) {
#pragma unroll
                for (int q = 0; q < Q; ++q) acc[q] = fmaf(dgs[item_n[q] * G + gg], Ws[gg * H + item_j[q]], acc[q]);
            }
            __syncthreads();
#pragma unroll
            for (int q = 0; q < Q; ++q) dhr[item_n[q] * H + item_j[q]] = acc[q];
        }
        __syncthreads();
    }
}

// dgin[row][frame][c] = sum over windows k covering `frame` of dgin_w[row*n_win + k][frame - k*stride][c]  (frames < T only)
__global__ void __launch_bounds__(256) lstm_fold_kernel(const float* __restrict__ dgin_w, float* __restrict__ dgin, int rows, int T,
                                                        int n_win, int steps, int stride, int C) {
    const int64_t total = (int64_t)rows * T * (C / 4);
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int c4 = (int)(i % (C / 4));
        const int64_t rf = i / (C / 4);
        const int frame = (int)(rf % T), row = (int)(rf / T);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        const int k_hi = min(n_win - 1, stride > 0 ? frame / stride : 0);
        for (int k = k_hi; k >= 0; --k) {
            const int pos = frame - k * stride;
            if (pos >= steps) break;
            const float4 v = reinterpret_cast<const float4*>(dgin_w + (((int64_t)row * n_win + k) * steps + pos) * C)[c4];
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        reinterpret_cast<float4*>(dgin + rf * C)[c4] = acc;
    }
}

template <int H, int NT>
static int launch_lstm_train_fwd(const float* gin, const float* bias_pad, const float* whh, float* hout, float* gates_s, float* c_s,
                                 float* h_s, const aero_lstm_params& p, cudaStream_t st) {
    const size_t smem = sizeof(float) * ((size_t)H * 4 * H + (size_t)H * NT + (size_t)NT * 4 * H);
    dim3 grid(cdiv(p.rows * p.n_win, NT), 2);
    cudaFuncSetAttribute(lstm_train_fwd_kernel<H, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    lstm_train_fwd_kernel<H, NT><<<grid, 4 * H, smem, st>>>(gin, bias_pad, whh, hout, gates_s, c_s, h_s, p);
    return check_launch("aero_lstm_train_fwd");
}

template <int H, int NT>
static int launch_lstm_bwd(const float* dhout, const float* gates_s, const float* c_s, const float* whh, float* dgin_w,
                           const aero_lstm_params& p, cudaStream_t st) {
    const size_t smem = sizeof(float) * ((size_t)4 * H * H + (size_t)NT * 4 * H + (size_t)NT * H);
    dim3 grid(cdiv(p.rows * p.n_win, NT), 2);
    cudaFuncSetAttribute(lstm_bwd_kernel<H, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    lstm_bwd_kernel<H, NT><<<grid, 4 * H, smem, st>>>(dhout, gates_s, c_s, whh, dgin_w, p);
    return check_launch("aero_lstm_bwd");
}

// Sequences per CTA: 16 when that still gives every SM a CTA, else fewer -- a training batch has a few hundred windows, and a CTA's step
// time is dominated by streaming W_hh from shared memory whatever NT is, so spreading the windows over more SMs is nearly free.
static int pick_nt(const aero_lstm_params& p, int nt_max) {
    static int num_sms = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    const int n_seq = p.rows * p.n_win;
    int nt = nt_max;
    while (nt > 4 && cdiv(n_seq, nt) * 2 < num_sms) nt >>= 1;
    return nt;
}

#define AERO_LSTM_NT_DISPATCH(FN, H_, NTMAX, ...)                          \
    switch (pick_nt(*p, NTMAX)) {                                          \
        case 16: return FN<H_, (NTMAX >= 16 ? 16 : NTMAX)>(__VA_ARGS__);   \
        case 8: return FN<H_, 8>(__VA_ARGS__);                             \
        default: return FN<H_, 4>(__VA_ARGS__);                            \
    }

}  // namespace aero

extern "C" int aero_lstm_train_fwd(const float* gin, const float* bias_pad, const float* whh, float* hout, float* gates_s, float* c_s,
                                   float* h_s, const aero_lstm_params* p, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(gin && whh && gates_s && c_s && h_s && p, "aero_lstm_train_fwd: null argument");
    AERO_REQUIRE(p->rows >= 1 && p->T >= 1 && p->n_win >= 1 && p->steps >= 1, "aero_lstm_train_fwd: bad sizes");
    AERO_REQUIRE(p->in_windowed || bias_pad, "aero_lstm_train_fwd: bias_pad required for un-windowed input");
    AERO_REQUIRE(p->out_windowed || hout, "aero_lstm_train_fwd: hout required for the de-windowed output");
    AERO_REQUIRE(p->n_win == 1 || (p->win_stride >= 2 && p->win_stride % 2 == 0), "aero_lstm_train_fwd: win_stride");
    cudaStream_t st = (cudaStream_t)stream;
    switch (p->H) {
        case 12: AERO_LSTM_NT_DISPATCH(launch_lstm_train_fwd, 12, 16, gin, bias_pad, whh, hout, gates_s, c_s, h_s, *p, st)
        case 24: AERO_LSTM_NT_DISPATCH(launch_lstm_train_fwd, 24, 16, gin, bias_pad, whh, hout, gates_s, c_s, h_s, *p, st)
        case 48: AERO_LSTM_NT_DISPATCH(launch_lstm_train_fwd, 48, 16, gin, bias_pad, whh, hout, gates_s, c_s, h_s, *p, st)
        case 96: AERO_LSTM_NT_DISPATCH(launch_lstm_train_fwd, 96, 16, gin, bias_pad, whh, hout, gates_s, c_s, h_s, *p, st)
        default:
            set_error("aero_lstm_train_fwd: hidden size %d not instantiated (12, 24, 48, 96)", p->H);
            return AERO_ERR_UNSUPPORTED;
    }
}

extern "C" int aero_lstm_bwd(const float* dhout, const float* gates_s, const float* c_s, const float* whh, float* dgin_w,
                             const aero_lstm_params* p, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(dhout && gates_s && c_s && whh && dgin_w && p, "aero_lstm_bwd: null argument");
    AERO_REQUIRE(p->rows >= 1 && p->T >= 1 && p->n_win >= 1 && p->steps >= 1, "aero_lstm_bwd: bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    switch (p->H) {
        case 12: AERO_LSTM_NT_DISPATCH(launch_lstm_bwd, 12, 16, dhout, gates_s, c_s, whh, dgin_w, *p, st)
        case 24: AERO_LSTM_NT_DISPATCH(launch_lstm_bwd, 24, 16, dhout, gates_s, c_s, whh, dgin_w, *p, st)
        case 48: AERO_LSTM_NT_DISPATCH(launch_lstm_bwd, 48, 16, dhout, gates_s, c_s, whh, dgin_w, *p, st)
        case 96: AERO_LSTM_NT_DISPATCH(launch_lstm_bwd, 96, 8, dhout, gates_s, c_s, whh, dgin_w, *p, st)
        default:
            set_error("aero_lstm_bwd: hidden size %d not instantiated (12, 24, 48, 96)", p->H);
            return AERO_ERR_UNSUPPORTED;
    }
}

extern "C" int aero_lstm_fold(const float* dgin_w, float* dgin, int32_t rows, int32_t T, int32_t n_win, int32_t steps, int32_t win_stride,
                              int32_t C, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(dgin_w && dgin && rows >= 1 && T >= 1 && n_win >= 1 && steps >= 1 && C % 4 == 0, "aero_lstm_fold: bad argument");
    AERO_REQUIRE(n_win == 1 || win_stride >= 1, "aero_lstm_fold: win_stride");
    const int64_t total = (int64_t)rows * T * (C / 4);
    int64_t blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    lstm_fold_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(dgin_w, dgin, rows, T, n_win, steps, win_stride, C);
    return check_launch("aero_lstm_fold");
}
