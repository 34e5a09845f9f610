/*
 * aero_b200.h -- C ABI of libaero_b200.so: the sm_90a kernels behind the AERO generator forward.
 *
 * The reference (slp-rl/aero) has no FFI: its hot path is the Python class
 * src/models/aero.py:218 `Aero`, whose arithmetic is dispatched to PyTorch library kernels.
 * Each entry point below replaces the library call(s) made at the cited reference lines.  A
 * binding needs nothing but device pointers, plain-old-data parameter blocks and a CUDA stream:
 * no ATen / Python types cross this boundary (see INTEGRATION.md for the ctypes stub).
 *
 * Conventions
 *   - All tensors are fp32, device memory, owned by the caller.  Kernels never allocate, never
 *     synchronise, and enqueue on `stream` only; entry points are re-entrant per stream.
 *   - Activations are channels-last: X[b][f][t][c] ("rows" (b,f) of T frames of C channels),
 *     the natural layout for this model (SURVEY.md 7.3): complex64 [B,F,T] *is* [B,F,T,2].
 *   - Return value: 0 on success, negative aero_status on error; aero_last_error() gives the
 *     text for the calling thread.  Launch errors are reported, asynchronous faults surface at
 *     the caller's next synchronisation.
 *   - Statistics buffers are fp64 pairs {sum, sum of squares} accumulated with atomics; the
 *     caller zeroes them (cudaMemsetAsync) before the producing call.
 */
#ifndef AERO_B200_H
#define AERO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* aero_stream_t; /* cudaStream_t */

enum aero_status {
    AERO_OK = 0,
    AERO_ERR_INVALID = -1,   /* bad parameter block */
    AERO_ERR_UNSUPPORTED = -2,
    AERO_ERR_LAUNCH = -3,    /* cudaGetLastError() after launch */
    AERO_ERR_NO_DEVICE = -4
};

int aero_abi_version(void);            /* 3: training entry points */
const char* aero_last_error(void);
/* compute capability of the current device as 10*major+minor (90 on H100); <0 if no device */
int aero_device_arch(void);
/* number of kernel launches issued through this library by the calling process (bench.py's gpu_launches) */
uint64_t aero_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * STFT  (replaces torch.stft at reference src/models/spec.py:12-20, called from aero.py:420,
 *        plus the Nyquist drop aero.py:420 `[..., :-1, :]`, the complex->channels permute
 *        aero.py:430-434 and the moments for aero.py:462-463)
 * x      : [n_signals][length]           real input, n_signals = B * channels
 * window : [win]                         analysis window (torch.hann_window(win), spec.py:15)
 * z      : element (sig, k, t) is the float2 at  z + (sig / channels) * z_stride_b
 *              + (sig % channels) * z_stride_c + k * z_stride_k + t * z_stride_t   (strides in floats)
 * stats  : optional [B][2] fp64 {sum, sumsq} over every float written for batch item b
 * Semantics: centre=True reflect padding of n_fft/2, window zero-padded (centred) to n_fft,
 * normalized=True (x n_fft^-1/2), onesided; bins 0 .. bins_out-1 are written
 * (bins_out = n_fft/2 drops Nyquist, n_fft/2+1 keeps it).  frames must equal 1 + length / hop.
 */
typedef struct {
    int32_t n_fft, hop, win;
    int32_t n_signals, channels;
    int32_t length, frames, bins_out;
    int64_t z_stride_b, z_stride_c, z_stride_k, z_stride_t;
    int32_t flags;                    /* 0, or AERO_STFT_* (training: this kernel is also the adjoint of the iSTFT) */
    int32_t reserved;
} aero_stft_params;
enum {
    AERO_STFT_ZERO_PAD = 1,           /* samples outside [0, length) are zero instead of reflected */
    AERO_STFT_ADJ_SCALE = 2           /* bins 1 .. n_fft/2-1 are doubled and the imaginary parts of DC / Nyquist zeroed: with ZERO_PAD and
                                         x = dy / envelope (zero-extended to hop*(frames-1)) this is dL/dz of aero_istft_fwd */
};
int aero_stft_fwd(const float* x, const float* window, float* z, double* stats,
                  const aero_stft_params* p, aero_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * iSTFT (replaces torch.istft at reference src/models/spec.py:30-37, called from aero.py:427,
 *        plus the Nyquist zero-pad aero.py:426 and the trim aero.py:513)
 * z addressing as above (bins_in bins present; bins above are taken as zero).
 * y : [n_signals][out_len],  y[n] = OLA(irfft(z * sqrt(n_fft)) * window)[n + n_fft/2] / sum(window^2)
 * out_len <= hop * (frames - 1).
 */
typedef struct {
    int32_t n_fft, hop, win;
    int32_t n_signals, channels;
    int32_t frames, bins_in, out_len;
    int64_t z_stride_b, z_stride_c, z_stride_k, z_stride_t;
    int32_t flags;                    /* 0, or AERO_ISTFT_RAW */
    int32_t reserved;
} aero_istft_params;
enum {
    AERO_ISTFT_RAW = 1                /* y[pos] = OLA(irfft(z * sqrt(n_fft)) * window)[pos], pos < out_len <= hop*(frames-1) + n_fft: no centre
                                         trim and no envelope division.  Applied to dL/dz with the interior bins halved this is the
                                         gradient of the reflect-PADDED input of aero_stft_fwd (the caller folds the padding back). */
};
int aero_istft_fwd(const float* z, const float* window, float* y,
                   const aero_istft_params* p, aero_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Tap-GEMM: every convolution / linear layer of the model as one implicit GEMM
 *   acc[b][fo][t][n] = sum_{tap} sum_{c < C1+C2}  A(b, fi(tap,fo), ti(tap,t), c) * W[slab(tap,fo)][c][n]
 * with A read from up to two channels-last sources (channel concat, reference aero.py:195
 * `torch.cat([x, skip], 1)`); out-of-range fi / ti contribute zero (zero padding).
 *   mode AERO_TAPS_CONV  : fi = fo*stride_f + jf - pad_f,  ti = t + jt*dil_t - pad_t,
 *                          slab = jf*kt + jt                      (nn.Conv2d / nn.Conv1d / nn.Linear)
 *   mode AERO_TAPS_CONVT : fo' = fo + f_out_offset (row in the uncropped output),
 *                          jf in [0, kf/stride_f): kf_idx = fo' % stride_f + jf*stride_f,
 *                          fi = fo' / stride_f - jf,  slab = kf_idx  (nn.ConvTranspose2d [k,1]/[s,1])
 *   mode AERO_TAPS_MIX   : (precision 1 / 2 only) contraction over the ROW axis of a channels-last tensor, FTB's
 *                          `freq_fc` (modules.py:296,317-320):  out[b][n][m] = colscale[b][m] * sum_{k<C1} a1[b][k][m] * W[n][k],
 *                          m < T pixels (contiguous), a1 element (b,k,m) at a1 + b*a1_sb + k*a1_st + m, out element
 *                          at out + b*o_sb + n*o_st + m, colscale at colscale + b*cs_sb + m.  F_out = F_in = 1.
 * Replaces nn.Conv2d/ConvTranspose2d (aero.py:89,95,101,172,179), nn.Conv1d (modules.py:80-92,
 * 206,209,292), nn.Linear (modules.py:29,296) and their cuDNN/cuBLAS kernels.
 *
 * Epilogue, in order:  v = acc + bias[n];  v *= colscale[b][t][n]  (FTB gate, modules.py:314);
 *   act (none | exact GELU | ReLU | LeakyReLU(0.2) | tanh);
 *   GLU over adjacent column pairs (2j, 2j+1) -> channel j  (weights are stored pair-interleaved);
 *   v += addend_fn[fo][n'] (frequency embedding, aero.py:475-480);
 *   v = residual[b][fo][t][n'] + v  ;  v = v * samp_affine[b][0] + samp_affine[b][1] (aero.py:497-498);
 *   statistics of the stored value:  stats_mode 1: per (b, group), group = n' / (N' / groups);
 *   stats_mode 2: per (b, fo) row.   N' = N/2 with GLU, else N.
 * Generic strides (in elements) let one kernel serve NCHW-free layouts: element (b,f,t,c) of a
 * source is at  src + b*sb + f*sf + t*st + c.
 */
enum { AERO_TAPS_CONV = 0, AERO_TAPS_CONVT = 1, AERO_TAPS_MIX = 2 };
enum { AERO_ACT_NONE = 0, AERO_ACT_GELU = 1, AERO_ACT_RELU = 2,
       AERO_ACT_LEAKY = 3 /* LeakyReLU(0.2); wgmma path: without residual or statistics */,
       AERO_ACT_TANH = 4 /* SIMT path only (aero_tapgemm_tc_eligible() is 0) */ };
typedef struct {
    int32_t B, F_out, T, N;
    int32_t F_in, T_in;
    int32_t C1, C2;
    int32_t mode, kf, kt, stride_f, pad_f, dil_t, pad_t, f_out_offset;
    int32_t act, glu, stats_mode, groups;
    int64_t a1_sb, a1_sf, a1_st;
    int64_t a2_sb, a2_sf, a2_st;
    int64_t w_sb;                     /* weight batch stride (0: shared weights) */
    int64_t o_sb, o_sf, o_st;
    int64_t r_sb, r_sf, r_st;         /* residual strides */
    int64_t cs_sb, cs_st;             /* colscale strides */
    int32_t precision;                /* 0: fp32 SIMT tiles, fp32 weights N-contiguous  W[slab][K][pad4(N)] (sources / outputs of either type);
                                         1: wgmma kind::tf32, fp32 sources, fp32 weights K-contiguous W[slab][pad4(N)][K] rounded to TF32;
                                         2: wgmma kind::f16, FP16 sources, FP16 weights K-contiguous W[slab][pad4(N)][pad8(K)];
                                            1 / 2: AERO_ERR_UNSUPPORTED unless aero_tapgemm_tc_eligible() */
    int32_t flags;                    /* AERO_TG_* */
} aero_tapgemm_params;
/* Storage types.  Activations that feed a tensor-core GEMM are stored either as fp32 rounded to TF32 or as FP16 (the same
 * 10-bit mantissa at half the bytes; stores saturate at +-65504); every kernel computes in fp32 between load and store.
 * Strides are in ELEMENTS of the tensor they address. */
enum {
    AERO_TG_ROUND_TF32 = 1,           /* fp32 outputs: round stored values to TF32 (round-to-nearest) for a kind::tf32 consumer */
    AERO_TG_A_F16 = 2,                /* a1 / a2 are FP16 */
    AERO_TG_OUT_F16 = 4,              /* out and residual are FP16 */
    AERO_TG_REVERSE = 8               /* tap-GEMM (wgmma path) / norm_act: walk tiles / rows from the end.  Results are identical;
                                         a kernel launched right after its producer then starts on the data the producer wrote last,
                                         which is still in the 50 MB L2 (the host alternates the direction from launch to launch) */
};
int aero_tapgemm_fwd(const void* a1, const void* a2, const void* w, const float* bias,
                     const float* addend_fn, const float* colscale, const void* residual,
                     const float* samp_affine, void* out, double* stats,
                     const aero_tapgemm_params* p, aero_stream_t stream);
/* 1 when the shape can run on the wgmma path (kind::tf32, or kind::f16 when flags has AERO_TG_A_F16), else 0 */
int aero_tapgemm_tc_eligible(const aero_tapgemm_params* p);

/* ------------------------------------------------------------------------------------------
 * Normalisation / activation passes (HBM-bound elementwise kernels)
 *
 * aero_sample_norm_fwd: per-sample standardisation of the input spectrogram (reference
 *   aero.py:462-464): mean / unbiased std over `count` values from stats[b] = {sum, sumsq};
 *   y = (x - mean) / (1e-5 + std) applied to `extent` (>= count; 0 means count) contiguous floats per sample -- rows may
 *   carry alignment padding that the statistics did not see; also writes samp_affine[b] = {std, mean} for the output
 *   de-normalisation (aero.py:497-498).
 */
int aero_sample_norm_fwd(const float* x, const double* stats, float* y, float* samp_affine,
                         int32_t B, int64_t count, int64_t extent, int32_t round_tf32, aero_stream_t stream);

/* aero_norm_act_fwd: y = op(GroupNorm(x))   (replaces nn.GroupNorm + F.gelu / F.glu / Snake /
 *   LayerScale + residual: aero.py:127,133,198,206-214; modules.py:189,210,232-244; snake.py:67)
 * x : [B][F_in][T][C]; rows f_off .. f_off+F_out-1 are read (decoder crop, aero.py:209).
 * stats : fp64 {sum, sumsq}; scope 1: [B][groups] over F_in*T*(C/groups) values (uncropped);
 *         scope 2: [B*F_in][1] per row over T*C values (DConv's GroupNorm(1, C)).
 * op: AERO_NA_NONE y=g; AERO_NA_GELU; AERO_NA_RELU y=max(g, 0); AERO_NA_GLU y[c]=g[c]*sigmoid(g[c+C/2]) (C_out=C/2);
 *     AERO_NA_SNAKE y = g + sin(a[f]*g)^2 / a[f];
 *     AERO_NA_GLU_SCALE_RES y[c] = residual[c] + scale[c] * glu(g)[c].
 */
enum { AERO_NA_NONE = 0, AERO_NA_GELU = 1, AERO_NA_GLU = 2, AERO_NA_SNAKE = 3, AERO_NA_GLU_SCALE_RES = 4,
       AERO_NA_RELU = 5, AERO_NA_LEAKY = 6 /* LeakyReLU(0.2) */, AERO_NA_TANH = 7 /* 6-7: training entry points only */ };
enum { AERO_NA_NO_NORM = 16 };      /* aero_norm_act_params.flags, training entry points: skip the normalisation (activation only) */
typedef struct {
    int32_t B, F_in, F_out, f_off, T, C;
    int32_t groups, scope, op;
    float eps;
    int32_t flags;                    /* AERO_TG_ROUND_TF32: round stored fp32 outputs to TF32 for a tensor-core consumer;
                                         AERO_TG_OUT_F16: y and residual are FP16; AERO_TG_A_F16: x is FP16 too (pre-normalisation
                                         tensors stored in FP16; the statistics were taken from the stored values); x == y is
                                         allowed when they have the same type and the op keeps the channel count */
} aero_norm_act_params;
int aero_norm_act_fwd(const void* x, const double* stats, const float* gamma, const float* beta,
                      const float* snake_a, const float* scale, const void* residual, void* y,
                      const aero_norm_act_params* p, aero_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * FTB output conv through a linear input (encoder layer 0: `pre_conv` aero.py:89,112 followed by FTB modules.py:304-325).
 * x = pre_conv(z) is linear in the J = 2*C_in spectrogram channels, and so is everything FTB does before its last ReLU:
 *   out[b,f,t,n] = relu( sum_{j<J} M[b,t][n][j] * zm[b,f,t,j] + M[b,t][n][J] * s[f] + sum_{j<J} V[n][j] * z[b,f,t,j] + d[n] )
 * with zm = freq_fc applied to z (AERO_TAPS_MIX), s[f] = sum_f' Wfc[f][f'], M[b,t] = gate[b,t,:] . Q,
 *   Q[c][n*(J+1)+j] = W2a[n][c] * (j < J ? Wpre[c][j] : bpre[c]),  V = W2b Wpre,  d = W2b bpre + b2
 * (W2 = [W2a | W2b] the BatchNorm-folded FTB conv2 acting on cat([freq_fc out, x]), modules.py:322-324).
 * z, zm : fp32, element (b,f,t,j) at base + b*sb + f*sf + t*J + j;  M : fp32 [B*T][N*(J+1)];  out : [B][F][T][N] fp32 / FP16.
 * The C-channel tensors pre_conv(z), freq_fc(..) and their concatenation are never materialised.
 */
typedef struct {
    int32_t B, F, T, N, J;
    int32_t flags;                    /* AERO_TG_OUT_F16 / AERO_TG_ROUND_TF32 */
    int64_t z_sb, z_sf, zm_sb, zm_sf;
} aero_ftb_lin_params;
int aero_ftb_lin_out_fwd(const float* z, const float* zm, const float* M, const float* s, const float* V, const float* d,
                         void* out, const aero_ftb_lin_params* p, aero_stream_t stream);
/* FTB squeeze (modules.py:286-291,308-309: 1x1 conv C -> r, BatchNorm, ReLU, regrouped to [B][T][F*r]) through the same
 * linearity:  R[b][t][f*r + n] = relu( sum_j W1p[n][j] * z[b,f,t,j] + b1p[n] ),  W1p = W1 Wpre [r][J], b1p = W1 bpre + b1, r <= 8.
 * R is fp32 or FP16 (flags); p->N is unused. */
int aero_ftb_lin_squeeze_fwd(const float* z, const float* W1p, const float* b1p, void* R, int32_t r,
                             const aero_ftb_lin_params* p, aero_stream_t stream);

/* FTB frequency mix (`freq_fc`, modules.py:296,317-320) for the deep layers where only F = 8 / 16 frequency rows are left:
 *   out[b][g][m] = gate[b][m] * sum_f W[g][f] * x[b][f][m],  m < M = T*C contiguous positions (M a multiple of 4), W fp32 [F][F],
 * gate fp32 [B][M] or NULL; x and out are both fp32 or both FP16 (AERO_TG_A_F16 | AERO_TG_OUT_F16).  Same result as
 * AERO_TAPS_MIX, without tensor-core tiles (they are all overhead at this F). */
int aero_freq_mix_small_fwd(const void* x, const float* W, const float* gate, void* out, int32_t B, int32_t F, int64_t M,
                            int32_t flags, aero_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Recurrent half of one bidirectional LSTM layer (replaces the cuDNN RNN behind nn.LSTM,
 * reference modules.py:28,46, together with the overlapping-window framing modules.py:36-44,
 * utils.py:22-35 and the central-crop reassembly modules.py:49-60).
 * The input projections x_t W_ih^T + b_ih + b_hh for BOTH directions are computed beforehand by
 * aero_tapgemm_fwd into `gin` (8H columns: [dir][i,f,g,o][H]).
 *   in_windowed = 0 : gin is [rows][T][8H] over the un-windowed sequence; window k, step p reads
 *                     frame k*win_stride + p; frames >= T are zero inputs, so their gate
 *                     pre-activation is `bias_pad` ([8H] = b_ih + b_hh)   (first layer)
 *   in_windowed = 1 : gin is [rows*n_win][steps][8H]                        (second layer)
 *   out_windowed = 1: h written as [rows*n_win][steps][2H]                  (first layer)
 *   out_windowed = 0: h written de-windowed as [rows][T][2H], keeping for window k the steps
 *                     [keep_lo(k), keep_hi(k)) exactly as modules.py:53-59    (second layer)
 * whh : [2][4H][H] (PyTorch layout weight_hh_l{k}, weight_hh_l{k}_reverse), gate order i,f,g,o.
 */
typedef struct {
    int32_t rows, T, H;
    int32_t n_win, steps, win_stride;
    int32_t in_windowed, out_windowed;
    int32_t flags;                    /* AERO_TG_ROUND_TF32: round the stored fp32 h to TF32; AERO_TG_OUT_F16: hout is FP16;
                                         AERO_TG_A_F16 (precision 1 only): gin is FP16 (bias_pad stays fp32) */
    int32_t precision;                /* 0: fp32 SIMT recurrence (layouts above);
                                         1: wgmma recurrence, FP16 operands (h in (-1,1), W_hh O(1): same 10-bit mantissa as TF32), fp32
                                            accumulate.  `gin` / `bias_pad` keep the layout above; only `whh` changes: FP16
                                            [2][(4/GPT)*128][Kp], Kp = 64*ceil(H/64), gate rows re-ordered into 4/GPT tiles of 128 per
                                            direction (GPT = 2 if H <= 64 else 1): GPT=1: tile g = gate g, row = cell; GPT=2: tile t =
                                            gates (2t, 2t+1), in each group of 32 rows rows 0-15 carry gate 2t and rows 16-31 gate 2t+1
                                            of the same 16 cells (zero rows beyond H, zero columns beyond H).  H % 4 == 0, 32 < H <= 96. */
} aero_lstm_params;
int aero_lstm_rec_fwd(const void* gin, const float* bias_pad, const void* whh, void* hout,
                      const aero_lstm_params* p, aero_stream_t stream);
/* Launch shape of the wgmma recurrence (precision 1) for n_seq = rows * n_win sequences on num_sms SMs: out[0] = sequences per
 * group (two groups per CTA), out[1] = wgmma N (8 or 16), out[2] = CTAs per direction, out[3] = cell-update threads per sequence.  AERO_ERR_INVALID outside the supported H. */
int aero_lstm_tc_shape(int32_t n_seq, int32_t H, int32_t num_sms, int32_t* out);

/* ------------------------------------------------------------------------------------------
 * LocalState attention core (replaces the einsum/softmax/einsum chain reference
 * modules.py:104-124; never materialises the T x T matrices).
 * qkvd : [rows][T][ld]  columns: q [0,H) | k [H,2H) | v (content) [2H,3H) | decay logits [3H, 3H+heads*ndecay)
 * out  : [rows][T][H],  out[s][h*d+c] = sum_t softmax_t( k_t.q_s/sqrt(d) - |t-s|*slope_s, diag=-100 ) * v_t[c]
 *        slope_s = sum_{f=1..ndecay} f * sigmoid(decay[h*ndecay+f-1][s]) / 2 / sqrt(ndecay)
 */
typedef struct {
    int32_t rows, T, H, heads, ndecay, ld;
    int32_t flags;                    /* AERO_TG_ROUND_TF32: tensor-core mode -- QK^T and PV on mma.sync TF32 (fp32 accumulate, head dim
                                         12 / 24), outputs rounded to TF32 for the projection GEMM; without it the exact fp32 SIMT kernel.
                                         AERO_TG_OUT_F16: out is FP16 */
} aero_attn_params;
int aero_local_attn_fwd(const float* qkvd, void* out, const aero_attn_params* p, aero_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Log-spectral distance (SURVEY.md section 8f rank 4; reference src/metrics.py:37-70 `get_lsd`, STFTMag(2048, 512)).
 * z_ref, z_est : planar complex spectrograms [B][bins][frames] (float2) as written by aero_stft_fwd (normalized);
 * out_sum += sum over (b, t) of sqrt(mean_f (log10 max(n_fft|z_ref|^2, 1e-8) - log10 max(n_fft|z_est|^2, 1e-8))^2).
 * The caller zeroes out_sum and divides by B * frames.
 */
int aero_lsd_fwd(const float* z_ref, const float* z_est, double* out_sum, int32_t B, int32_t bins, int32_t frames,
                 int32_t n_fft, aero_stream_t stream);

/* aero_lsd_varlen_fwd: the same distance fused with its STFTs (n_fft 2048, hop 512, periodic Hann, centred, not normalised)
 * for rows of different lengths, one value per file.
 * ref, est      : waveforms [rows][L_max] (fp32); row r holds lengths[r] valid samples (1024 < lengths[r] <= L_max) and is
 *                 reflect padded by 1024 at its own two ends; samples past lengths[r] are never read.
 * row_file      : file of each row, in [0, n_files); every file has at least one row.
 * row_frame_off : [rows + 1] first frame of each row in frame_lsd; row r has 1 + lengths[r] / 512 frames, at most max_frames.
 * frame_lsd     : workspace [row_frame_off[rows]], the per-frame distances (fp32).
 * out           : [n_files] fp32, the mean over all frames of all rows of each file, summed in fp64 in a fixed order.
 * Two launches, no atomics: each file's value depends only on its own rows, bit for bit.
 */
int aero_lsd_varlen_fwd(const float* ref, const float* est, int32_t rows, int32_t L_max, const int32_t* lengths,
                        const int32_t* row_file, const int32_t* row_frame_off, int32_t max_frames, int32_t n_files,
                        float* frame_lsd, float* out, aero_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Multi-resolution STFT loss, forward value (SURVEY.md section 8f rank 2; reference src/models/stft_loss.py:11-27,30-63,96-138).
 * z_est, z_ref : planar complex spectrograms [B][bins][frames] (float2) of the estimate and the target as written by
 * aero_stft_fwd (normalised) at ONE resolution; with mag = sqrt(max(n_fft |z|^2, 1e-7)):
 *   sums[0] += sum (mag_ref - mag_est)^2;  sums[1] += sum mag_ref^2;  sums[2] += sum |log mag_ref - log mag_est|
 * -> spectral convergence = sqrt(sums[0]/sums[1]), log-magnitude L1 = sums[2] / (B*bins*frames).  The caller zeroes `sums`.
 */
int aero_stft_loss_fwd(const float* z_est, const float* z_ref, double* sums, int32_t B, int32_t bins, int32_t frames,
                       int32_t n_fft, aero_stream_t stream);

/* Backward of the above for the estimate: with the `sums` of the forward, g_est[B][bins][frames] (float2) = gradient of
 *   c_sc * sqrt(sums[0]/sums[1]) + c_mag * sums[2] / (B*bins*frames)
 * with respect to the normalised spectrogram z_est, the interior bins already halved: feeding g_est to aero_istft_fwd with
 * AERO_ISTFT_RAW gives the gradient of the reflect-padded waveform (the caller folds the padding back).  bins = n_fft/2+1.
 * (reference: autograd through stft_loss.py:11-63, called with gradients at solver.py:470-473) */
int aero_stft_loss_bwd(const float* z_est, const float* z_ref, const double* sums, float* g_est, int32_t B, int32_t bins,
                       int32_t frames, int32_t n_fft, float c_sc, float c_mag, aero_stream_t stream);

/* ==========================================================================================
 * Training (SURVEY.md section 8f rank 1: backward of the custom ops + fused Adam; reference callers src/solver.py:292-342,
 * 602-605 `loss.backward(); optimizer.step()`, train.py:83 `torch.optim.Adam`).  All tensors fp32.
 *
 * Data gradients of every convolution / linear layer run on aero_tapgemm_fwd itself: the adjoint of a tap-GEMM is a
 * tap-GEMM (taps flipped, weights transposed, AERO_TAPS_CONV <-> AERO_TAPS_CONVT for strided layers).
 * ========================================================================================== */

/* Weight gradient of a tap-GEMM:  dW(n, k, slab) += sum_{b,fo,t} A(b, fi, ti, k) * dY(b, fo, t, n)  with (fi, ti, slab) the tap
 * geometry of aero_tapgemm_fwd for `p` (mode AERO_TAPS_CONV or AERO_TAPS_CONVT; A = channel concat of a1, a2).  dY is addressed
 * with p->o_sb / o_sf / o_st; element (n, k, slab) of dW lives at dw + n*dw_sn + k*dw_sk + slab*dw_ss (so the gradient can be
 * written straight into PyTorch's [N][K][kf][kt] or ConvTranspose [K][N][kf][1] parameter layout).  The caller zeroes dW.
 * p->precision: 0 = exact fp32 (SIMT; a one-thread-per-weight kernel when the layer has at most 2048 weights); 1 = TF32 on the
 * tensor cores (csrc/wgrad_tc.cu: both operands MN-major through TMA, split over the pixel axis, fp32 atomics) where the shape allows
 * (N >= 16, K >= 16, channel counts and strides multiples of 4, 16-byte aligned bases), exact fp32 otherwise.
 * Replaces the cuDNN wgrad kernels behind autograd of nn.Conv2d / ConvTranspose2d / Conv1d / Linear. */
int aero_tapgemm_wgrad(const float* a1, const float* a2, const float* dy, float* dw, const aero_tapgemm_params* p,
                       int64_t dw_sn, int64_t dw_sk, int64_t dw_ss, aero_stream_t stream);

/* Column sums:  out1[seg][n] += sum_{o < n_outer, i < n_inner} x[seg*seg_stride_x + o*outer_stride + i*inner_stride + n],
 * out2[seg][n] += the same sum of x * z (z addressed like x; NULL: skipped).  out_double: outputs are fp64 (statistics) else fp32.
 * Bias gradients, BatchNorm batch statistics (z = x), frequency-embedding gradients.  The caller zeroes the outputs. */
int aero_colsum(const float* x, const float* z, void* out1, void* out2, int32_t out_double, int32_t N, int64_t n_inner,
                int64_t inner_stride, int64_t n_outer, int64_t outer_stride, int32_t n_seg, int64_t seg_stride_x,
                int64_t seg_stride_out, aero_stream_t stream);

/* out[i][j] += sum_{b, m} P[b][i][m] * gate[b][m] * Q[b][j][m],  i, j < F,  m < M contiguous (batch strides sb_*; gate may be
 * NULL): weight gradient of FTB's `freq_fc` (modules.py:296,317-320), P = dY, Q = x, gate = the FTB gate.  Caller zeroes out. */
int aero_gram(const float* P, const float* Q, const float* gate, float* out, int32_t B, int32_t F, int64_t M, int64_t sb_p,
              int64_t sb_q, int64_t sb_g, aero_stream_t stream);
/* x[b][f][t][c] += addend[f][c]  (frequency embedding, aero.py:475-480; fused into a GEMM epilogue at inference). */
int aero_bcast_add(float* x, const float* addend, int32_t B, int32_t F, int32_t T, int32_t C, aero_stream_t stream);
/* y[b][i] = x[b][i] * s[b*s_stride], i < per_sample  (backward of the per-sample de-normalisation aero.py:497-498). */
int aero_scale_rows(const float* x, float* y, const float* s, int32_t B, int64_t per_sample, int32_t s_stride, aero_stream_t stream);
/* dst[i] += alpha * src[i] (gradient accumulation where a tensor has several consumers). */
int aero_add(float* dst, const float* src, int64_t n, float alpha, aero_stream_t stream);
/* dst[i] += (float) src[i]: fp64 column sums into an fp32 parameter gradient. */
int aero_add_f64(float* dst, const double* src, int64_t n, aero_stream_t stream);

/* Normalisation + activation, training form (nothing folded, fp32): y = act(norm(x)) with
 *   scope 1 / 2: GroupNorm as in aero_norm_act_fwd;  scope 3: BatchNorm with BATCH statistics, stats = [C][2] fp64 {sum, sumsq}
 *   over all B*F_in*T pixels (reference modules.py:287-300 in train mode);  flags & AERO_NA_NO_NORM: activation only.
 * ops: AERO_NA_* (SNAKE needs scope 2).  x [B][F_in][T][C], y [B][F_out][T][C or C/2]. */
int aero_norm_act_train_fwd(const float* x, const double* stats, const float* gamma, const float* beta, const float* snake_a,
                            const float* scale, const float* residual, float* y, const aero_norm_act_params* p,
                            aero_stream_t stream);
/* Backward of the above.  pass 1 accumulates dgamma[C], dbeta[C], dscale[C/2] (GLU_SCALE_RES), dsnake[F_in] (SNAKE) -- all fp64:
 * these are sums over every pixel of the batch whose terms largely cancel, and fp32 atomics across hundreds of CTAs lose
 * ~1e-3 of the result -- and the per-(segment, group) sums ws[slot] = {sum dxh, sum dxh*xh} (fp64, same slots as `stats`;
 * unused for scope 3, which reads dgamma / dbeta instead);
 * pass 2 writes dx[B][F_in][T][C] = rstd * (dxh - mean(dxh) - xh * mean(dxh * xh)) (every input row, cropped rows included).
 * The gradient of the residual input of GLU_SCALE_RES is dy itself (the caller accumulates it).  The caller zeroes the
 * accumulators before pass 1. */
int aero_norm_act_train_bwd(const float* x, const double* stats, const float* gamma, const float* beta, const float* snake_a,
                            const float* scale, const float* dy, float* dx, double* dgamma, double* dbeta, double* dscale,
                            double* dsnake, double* ws, int32_t pass, const aero_norm_act_params* p, aero_stream_t stream);

/* LSTM layer, training form (fp32 SIMT recurrence; reference modules.py:28-65 under autograd, i.e. cuDNN's RNN training
 * forward and backward-data).  Forward = aero_lstm_rec_fwd (precision 0) that also saves, WINDOWED as [rows*n_win][steps][2][..],
 * the post-activation gates (i,f,g,o: 4H), the cell state c (H) and the hidden state h (H) of every step; hout is the
 * de-windowed output (may be NULL when out_windowed: h_s is that output).
 * Backward: dhout in the layout of the forward's output (windowed [n_seq][steps][2H] or de-windowed [rows][T][2H]);
 * dgin_w = gradient of the gate pre-activations, windowed [n_seq][steps][2][4H] (every position, padding frames included).
 * The caller finishes with GEMMs over dgin_w: bias = column sums, W_hh = aero_tapgemm_wgrad against h_s shifted by one step,
 * W_ih / input gradient from dgin (aero_lstm_fold sums the windowed rows back onto un-windowed frames for the first layer). */
int aero_lstm_train_fwd(const float* gin, const float* bias_pad, const float* whh, float* hout, float* gates_s, float* c_s,
                        float* h_s, const aero_lstm_params* p, aero_stream_t stream);
int aero_lstm_bwd(const float* dhout, const float* gates_s, const float* c_s, const float* whh, float* dgin_w,
                  const aero_lstm_params* p, aero_stream_t stream);
int aero_lstm_fold(const float* dgin_w, float* dgin, int32_t rows, int32_t T, int32_t n_win, int32_t steps, int32_t win_stride,
                   int32_t C, aero_stream_t stream);

/* LocalState attention, training form (reference modules.py:104-124 under autograd): exact-fp32 forward that also returns
 * lse[rows][heads][T] (log-sum-exp over keys per query), and the backward: dqkvd[rows][T][ld] (q | k | v | decay-logit columns,
 * every column written) from dout[rows][T][H]; scores are recomputed flash-style (no T x T tensor). */
int aero_local_attn_train_fwd(const float* qkvd, float* out, float* lse, const aero_attn_params* p, aero_stream_t stream);
int aero_local_attn_bwd(const float* qkvd, const float* out, const float* lse, const float* dout, float* dqkvd,
                        const aero_attn_params* p, aero_stream_t stream);

/* MelGAN multi-scale discriminator (SURVEY.md section 8f rank 3; reference src/models/discriminators.py:14-78): grouped strided
 * Conv1d (k <= 41, <= 8 input channels per group) on channels-last tensors x [B][Tin][Cin] -> y [B][Tout][Cout], weights in
 * PyTorch's layout w [Cout][Cin/groups][k]; Tout = (Tin + 2 pad - k) / stride + 1.  dgrad writes dx; wgrad ADDS into dw (caller zeroes).
 * The dense layers of the discriminator (k = 15 / 5 / 3) run on aero_tapgemm_fwd / aero_tapgemm_wgrad. */
int aero_gconv1d_fwd(const float* x, const float* w, const float* bias, float* y, int32_t B, int32_t Tin, int32_t Tout, int32_t Cin,
                     int32_t Cout, int32_t groups, int32_t k, int32_t stride, int32_t pad, aero_stream_t stream);
int aero_gconv1d_dgrad(const float* dy, const float* w, float* dx, int32_t B, int32_t Tin, int32_t Tout, int32_t Cin, int32_t Cout,
                       int32_t groups, int32_t k, int32_t stride, int32_t pad, aero_stream_t stream);
int aero_gconv1d_wgrad(const float* x, const float* dy, float* dw, int32_t B, int32_t Tin, int32_t Tout, int32_t Cin, int32_t Cout,
                       int32_t groups, int32_t k, int32_t stride, int32_t pad, aero_stream_t stream);
/* Weight normalisation (torch.nn.utils.weight_norm, reference modules.py WNConv1d): w[r][:] = g[r] * v[r][:] / ||v[r][:]||, and its
 * backward, which ADDS  dg[r] += <dw[r], v[r]> / ||v[r]||  and  dv[r] += g[r]/||v[r]|| * (dw[r] - v[r] <dw[r], v[r]> / ||v[r]||^2). */
int aero_weight_norm_fwd(const float* v, const float* g, float* w, int32_t rows, int32_t len, aero_stream_t stream);
int aero_weight_norm_bwd(const float* v, const float* g, const float* dw, float* dv, float* dg, int32_t rows, int32_t len,
                         aero_stream_t stream);

/* Weight repack for the tensor-core training modes: w [taps][K][ldn] (the aero_tapgemm_fwd precision-0 layout, ldn = N rounded up to
 * 4) -> out [taps][ldn][K] (the precision-1 layout), every element rounded to TF32 (round to nearest, ties away); out_lo (optional) gets
 * TF32(w - out) in the same layout.
 * aero_split_tf32: the same two-term split of an activation tensor, hi = TF32(x), lo = TF32(x - hi).  Three TF32 tensor-core products
 * hi*hi + hi*lo + lo*hi, summed in fp32, reproduce the fp32 product to ~2^-22 ("3xTF32"): the training engine's fp32-grade tensor-core
 * mode issues aero_tapgemm_fwd / aero_tapgemm_wgrad three times on these halves (aero_b200/train_engine.py, precision 3).
 * aero_tapgemm_wgrad_tc_eligible: 1 when aero_tapgemm_wgrad with p->precision = 1 would run on the tensor cores. */
int aero_pack_kmajor_tf32(const float* w, float* out, float* out_lo, int32_t taps, int32_t K, int32_t ldn, aero_stream_t stream);
int aero_split_tf32(const float* x, float* hi, float* lo, int64_t n, aero_stream_t stream);
int aero_tapgemm_wgrad_tc_eligible(const aero_tapgemm_params* p, const float* a1, const float* a2, const float* dy);

/* Fused multi-tensor Adam (torch.optim.Adam semantics, no amsgrad / weight decay; reference train.py:83).  chunk_table: device
 * array of n_chunks records {float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64 count}; one CTA per
 * record.  step >= 1 is the step count AFTER this update (bias corrections 1 - beta^step); grad_scale multiplies every
 * gradient (1/world_size after a sum all-reduce). */
int aero_adam_step(const void* chunk_table, int32_t n_chunks, float lr, float beta1, float beta2, float eps, int32_t step,
                   float grad_scale, aero_stream_t stream);

/* ==========================================================================================
 * SEANet generator (reference src/models/seanet.py), time domain, channels-last activations [B][frames][C].
 * ========================================================================================== */

/* Input stage (seanet.py:158-168): per clip, std = unbiased std over the L_in samples of the channel mean (fp64 sums; 1 when
 * normalize == 0), x' = x / (floor + std); then the polyphase Hann-windowed sinc resampler the reference calls (`up` phases of
 * `taps` fp32 coefficients filt[up][taps], input stride `orig`, left pad `width`; up == 0: no resampling, L_hr = L_in), then zero
 * padding to L_valid frames.  x : [B][C][L_in] fp32.  x0 : fp32, element (b, u, c) at x0 + b*(L_valid + 2*halo)*C + (halo + u)*C + c;
 * frames u in [-fill, L_valid + fill) are written, the ones outside [0, L_valid) by reflection (fill < L_valid, fill <= halo).
 * affine[b] = {std, 0}: the output scaling of seanet.py:179 as a tap-GEMM samp_affine. */
typedef struct {
    int32_t B, C, L_in;
    int32_t orig, up, width, taps;
    int32_t L_hr, L_valid, halo, fill;
    int32_t normalize;
    float floor_;
} aero_resample_params;
int aero_seanet_input_fwd(const float* x, const float* filt, float* affine, float* x0, const aero_resample_params* p,
                          aero_stream_t stream);

/* Hann-windowed sinc resampling (the reference's data-pipeline resampler with its default filter) of `rows` independent
 * signals: x [rows][L_in] -> y [rows][L_out], fp32,
 *   y[r][t] = sum_k filt[t % up][k] * x[r][(t / up) * orig - width + k]   (k < taps; x is zero outside [0, L_in)),
 * with filt[up][taps] the polyphase table of the reduced ratio orig:up (taps = 2*width + orig) and
 * L_out <= (L_in / orig + 1) * up (the reference keeps ceil(up * L_in / orig)).  The same per-sample filter as
 * aero_seanet_input_fwd. */
int aero_resample_fwd(const float* x, const float* filt, float* y, int64_t rows, int32_t L_in, int32_t L_out, int32_t orig, int32_t up,
                      int32_t width, int32_t taps, aero_stream_t stream);

/* Reflection halo + activation (nn.ReflectionPad1d after nn.LeakyReLU, seanet.py:14-16,58-59):
 *   y(b, u, c) = act(x(b, r(u), c)),  u in [-halo, T + halo),  r(u) = |u| reflected at both ends (halo < T),
 * x element (b, t, c) at x + b*x_sb + t*C + c, y element (b, u, c) at y + b*y_sb + u*C + c (y points at frame 0; the halo
 * frames lie before and after it).  act: AERO_ACT_NONE or AERO_ACT_LEAKY.  flags: AERO_TG_A_F16 (x FP16), AERO_TG_OUT_F16
 * (y FP16), AERO_TG_ROUND_TF32 (fp32 y rounded to TF32).  C % 4 == 0.  A consumer convolution at dilation d then reads frame
 * -d as its first input frame with no zero padding. */
int aero_reflect_act_fwd(const void* x, void* y, int32_t B, int32_t T, int32_t C, int64_t x_sb, int64_t y_sb, int32_t halo,
                         int32_t act, int32_t flags, aero_stream_t stream);

/* Training adjoint of aero_reflect_act_fwd (fp32):  dx(b, t, c) = act'(x(b, t, c)) * sum over u with r(u) = t of dy(b, u, c),
 * u in [-halo, T + halo): the halo's gradient folded back onto the mirrored frames.  dy element (b, u, c) at dy + b*dy_sb + u*C + c
 * (dy points at frame 0), dx [B][T][C] contiguous, x as in the forward (act' needs it; unused for AERO_ACT_NONE). */
int aero_reflect_act_bwd(const float* x, const float* dy, float* dx, int32_t B, int32_t T, int32_t C, int64_t x_sb, int64_t dy_sb,
                         int32_t halo, int32_t act, aero_stream_t stream);

/* SEANet output (seanet.py:116-118,176,179), training form: y[b][i] = affine[b][0] * (tanh(v[b][i]) + x0[b][i]), i < per_clip;
 * backward dv[b][i] = dy[b][i] * affine[b][0] * (1 - tanh(v[b][i])^2).  All fp32, contiguous per clip. */
int aero_seanet_output_fwd(const float* v, const float* x0, const float* affine, float* y, int32_t B, int64_t per_clip,
                           aero_stream_t stream);
int aero_seanet_output_bwd(const float* v, const float* affine, const float* dy, float* dv, int32_t B, int64_t per_clip,
                           aero_stream_t stream);

/* ==========================================================================================
 * HiFi-GAN multi-period discriminator (reference src/models/discriminators.py:89-147), fp32.  Each period's activations are one
 * long channels-last sequence of B*period segments s = b*period + w; segment s holds frames h of column w of the [T/period, period]
 * view at rows s*seg + halo + h, and zeros at every other row (see DESIGN.md, "Multi-period discriminator").
 * ========================================================================================== */

/* Period fold (discriminators.py:107-113): x [B][T] -> y [B*period][seg] with y[(b*period + w)*seg + halo + h] = xp[b][h*period + w],
 * h < H = ceil(T / period), where xp is x reflect-padded on the right to H*period samples (H*period - T < T); every other element of y
 * is written 0.  Backward: dx[b][t] = dy at the position of t + dy at the position of its mirror 2(T-1) - t when that lies in the
 * padding (the gradient that reaches the generator). */
int aero_mpd_fold_fwd(const float* x, float* y, int32_t B, int32_t T, int32_t period, int32_t H, int32_t seg, int32_t halo,
                      aero_stream_t stream);
int aero_mpd_fold_bwd(const float* dy, float* dx, int32_t B, int32_t T, int32_t period, int32_t H, int32_t seg, int32_t halo,
                      aero_stream_t stream);

/* Activation repack (LeakyReLU(slope) after each convolution, discriminators.py:116-118): x element (s, h, c) at
 * x[(s*rows_in + h)*C + c], h < H (a convolution's output rows; rows H .. rows_in-1 of a segment are ignored) ->
 * y[(s*seg + halo + h)*C + c] = leaky(x), every other element of y [S][seg][C] written 0, so that y is the next convolution's input.
 * Backward: dx[(s*rows_in + r)*C + c] = dy[(s*seg + halo + r)*C + c] * leaky'(x) for r < H and 0 for r >= H (every element of dx
 * written: rows no output frame owns carry no gradient into the weight and bias sums).  C % 4 == 0, pointers 16-byte aligned. */
int aero_mpd_repack_fwd(const float* x, float* y, int32_t S, int32_t H, int32_t C, int32_t rows_in, int32_t seg, int32_t halo,
                        float slope, aero_stream_t stream);
int aero_mpd_repack_bwd(const float* x, const float* dy, float* dx, int32_t S, int32_t H, int32_t C, int32_t rows_in, int32_t seg,
                        int32_t halo, float slope, aero_stream_t stream);

/* ==========================================================================================
 * GAN loss terms (reference src/solver.py:475-520, src/models/discriminators.py:211-244) on the discriminators' own storage.
 * A term is one feature map stored as n_seg segments of seg rows x C channels, channels-last: element (s, h, c) of the map sits at
 * x[(s*seg + halo + h)*C + c], h < H (the owned rows); the other rows of a segment belong to no output.  This is the MPD segment
 * layout and, with one segment per clip and halo 0, MelGAN's [B, T, C].  Its count is n = n_seg*H*C.
 * ========================================================================================== */

enum {
    AERO_GAN_NONE = 0,
    AERO_GAN_LSGAN_REAL = 1,   /* (1 - x)^2                        (discriminator, real clips)      */
    AERO_GAN_LSGAN_FAKE = 2,   /* x^2                              (discriminator, generated clips) */
    AERO_GAN_LSGAN_GEN = 3,    /* (1 - x)^2                        (generator)                      */
    AERO_GAN_HINGE_REAL = 4,   /* relu(1 - x)                      (discriminator, real clips)      */
    AERO_GAN_HINGE_FAKE = 5,   /* relu(1 + x)                      (discriminator, generated clips) */
    AERO_GAN_HINGE_GEN = 6     /* relu(1 - x)                      (generator)                      */
};

#define AERO_GAN_FWD_BLOCKS 128   /* blocks per term of aero_gan_loss_fwd: its workspace holds n_terms * 2 * this many doubles */

typedef struct {
    const float* x;      /* the map                                                                      */
    const float* ref;    /* L1 reference map of the same geometry (the real clips' features), or NULL    */
    float* dx;           /* gradient storage of x, n_seg*seg*C floats (aero_gan_loss_bwd)                */
    double adv_scale;    /* weight / count of the adversarial mean (0: no adversarial component)         */
    double l1_scale;     /* weight / count of the L1 mean (0 or ref NULL: no L1 component)               */
    int32_t n_seg, seg, halo, H, C;
    int32_t adv;         /* AERO_GAN_*                                                                   */
} aero_gan_term;

/* Forward of n_terms terms (terms: a DEVICE table) in one call: out[2t] = adv_scale * sum adv(x), out[2t + 1] =
 * l1_scale * sum |x - ref| over the owned elements of term t, in fp64.  Deterministic: per-block partial sums in a fixed order
 * (work: n_terms * 2 * AERO_GAN_FWD_BLOCKS doubles), then one fixed-order reduction per term; no floating-point atomics.  A term
 * whose geometry is invalid (n_seg, H or C < 1, halo < 0, halo + H > seg) yields NaN. */
int aero_gan_loss_fwd(const aero_gan_term* terms, int32_t n_terms, double* out, double* work, aero_stream_t stream);

/* Backward: writes every element of each term's dx -- owned elements get (float)adv_scale * adv'(x) + (float)l1_scale * sign(x - ref)
 * (fp32; relu' and sign are 0 at their kinks, as in PyTorch), every other row exact 0.  Terms may share a dx buffer only on
 * disjoint element ranges. */
int aero_gan_loss_bwd(const aero_gan_term* terms, int32_t n_terms, aero_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Ragged batches: clips of different lengths in one forward, each with the result it gets on its own.
 * Clip b occupies the first frames[b] frames of the usual [B][F][T][C] tensors (T = the batch's longest clip); the rest are
 * padding.  Padded frames are left out of every reduction and sequence op, and hold exact zeros in every tensor a
 * time-coupled convolution reads.  Length tables (`lengths`, `frames`, `out_lens`) are int32 DEVICE arrays with one entry per
 * clip.
 *
 * aero_stft_varlen_fwd: aero_stft_fwd for signals of lengths[b] valid samples in rows of p->length (a multiple of hop;
 *   p->frames = 1 + length/hop).  Each signal is zero padded to a multiple of hop and reflected at that padded end
 *   (reference aero.py:409-420, spec.py:9-22, on the clip alone); frames at or past its own 1 + padded/hop are written as
 *   zeros, and stats[b] accumulates {sum, sumsq} over its valid frames only.  p->flags must be 0.
 *   Preconditions (the caller's; they cannot be checked without reading the device table): 1 <= lengths[b] <= p->length and
 *   lengths[b] padded to a multiple of hop > n_fft/2 (reflect padding, as for aero_stft_fwd).  Out of contract, the kernel
 *   clamps lengths[b] to p->length and reads no sample outside the signal's row (such frames are garbage, not a fault).
 */
int aero_stft_varlen_fwd(const float* x, const float* window, float* z, double* stats, const int32_t* lengths,
                         const aero_stft_params* p, aero_stream_t stream);
/* aero_istft_varlen_fwd: aero_istft_fwd where signal b uses frames[b] frames and writes out_lens[b] samples of its row of
 *   p->out_len (the rest of the row is zeroed).  p->flags must be 0. */
int aero_istft_varlen_fwd(const float* z, const float* window, float* y, const int32_t* frames, const int32_t* out_lens,
                          const aero_istft_params* p, aero_stream_t stream);
/* aero_sample_norm_varlen_fwd: aero_sample_norm_fwd with each clip's own count, per_frame * frames[b] values; `extent`
 *   floats per sample are transformed. */
int aero_sample_norm_varlen_fwd(const float* x, const double* stats, float* y, float* samp_affine, const int32_t* frames,
                                int32_t B, int64_t per_frame, int64_t extent, int32_t round_tf32, aero_stream_t stream);
/* aero_masked_stats_fwd: GroupNorm statistics of a stored tensor x [B][F][T][C] (fp32, or FP16 with AERO_TG_A_F16) over
 *   the valid frames t < frames[b] only, added into the slots aero_norm_act_fwd reads (scope 1: [B][groups]; scope 2:
 *   [B*F]), scaled by T / frames[b] so that norm_act's count over T frames gives the clip's own mean and variance. */
int aero_masked_stats_fwd(const void* x, double* stats, const int32_t* frames, int32_t B, int32_t F, int32_t T, int32_t C,
                          int32_t groups, int32_t scope, int32_t flags, aero_stream_t stream);
/* aero_frame_mask_fwd: x [B][F][T][C] (fp32, or FP16 with AERO_TG_OUT_F16): frames t >= frames[b] are set to zero. */
int aero_frame_mask_fwd(void* x, const int32_t* frames, int32_t B, int32_t F, int32_t T, int32_t C, int32_t flags,
                        aero_stream_t stream);
/* aero_gather_rows_fwd: dst[i][c] = src[idx[i*parts + c/(width/parts)]][c] for rows of `width` elements (fp32, or FP16 with
 *   AERO_TG_A_F16); a negative index takes fill[c] (fp32; zero when fill is NULL).  The ragged BiLSTM uses it to lay each
 *   clip's sequences (its own step count, windows of reference modules.py:32-65 past 200 frames, bias-only input past its
 *   end, the reverse direction starting at its own last step) onto the windowed layout of aero_lstm_rec_fwd and back. */
int aero_gather_rows_fwd(const void* src, void* dst, const int32_t* idx, const float* fill, int64_t n_rows, int32_t width,
                         int32_t parts, int32_t flags, aero_stream_t stream);
/* aero_local_attn_varlen_fwd: aero_local_attn_fwd where row r belongs to clip r / rows_per_clip and only its first
 *   frames[clip] frames take part (keys, queries, decay, softmax); outputs of the padded frames are not written. */
int aero_local_attn_varlen_fwd(const float* qkvd, void* out, const int32_t* frames, int32_t rows_per_clip,
                               const aero_attn_params* p, aero_stream_t stream);
/* aero_seanet_input_varlen_fwd: aero_seanet_input_fwd where clip b holds lengths[b] valid samples in its rows of p->L_in
 *   samples.  p describes the buffers: p->L_hr and p->L_valid are those of a clip of p->L_in samples (the longest), and x0 has
 *   p->L_valid + 2*p->halo frames per clip.  Each clip gets what a single-clip call of its own length writes: std of its own
 *   lengths[b] samples (same fp64 summation order), resampled to hr_lengths[b] samples (samples at or past lengths[b] are
 *   never read), zero padded to valid_lengths[b] frames, `fill` frames reflected at both of its own ends, affine[b] = {std, 0}.
 *   Frames u in [valid_lengths[b] + fill, p->L_valid + p->halo) are written as zeros.
 *   Preconditions (the caller's; they cannot be checked without reading the device tables): 2 <= lengths[b] <= p->L_in,
 *   hr_lengths[b] = the resampled length of lengths[b] samples (= lengths[b] when p->up == 0), hr_lengths[b] <= valid_lengths[b]
 *   <= p->L_valid and p->fill < valid_lengths[b].  Out of contract, every table entry is clamped to the buffer and no sample
 *   outside the clip's row is read (such frames are garbage, not a fault). */
int aero_seanet_input_varlen_fwd(const float* x, const float* filt, float* affine, float* x0, const int32_t* lengths,
                                 const int32_t* hr_lengths, const int32_t* valid_lengths, const aero_resample_params* p,
                                 aero_stream_t stream);
/* aero_reflect_act_varlen_fwd: aero_reflect_act_fwd where clip b has frames[b] of the T frames (T = the longest clip's).  It
 *   writes act(x) on [0, frames[b]), the reflection at the clip's own ends on [-halo, 0) and [frames[b], frames[b] + halo), and
 *   zeros on [frames[b] + halo, T + halo); frames[b] and past of x are never read.  With halo = 0 this is the input of a
 *   zero-padded convolution (SEANet's strided and transposed convolutions over super-frames): the clip's frames are followed by
 *   exact zeros.  Preconditions: halo < frames[b] <= T.  Out of contract, frames[b] is clamped to T and no frame outside
 *   [0, T) of x is read. */
int aero_reflect_act_varlen_fwd(const void* x, void* y, const int32_t* frames, int32_t B, int32_t T, int32_t C, int64_t x_sb,
                                int64_t y_sb, int32_t halo, int32_t act, int32_t flags, aero_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* AERO_B200_H */
