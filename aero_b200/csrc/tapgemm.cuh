// Shared argument block of the tap-GEMM implementations.
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace aero {
struct TapGemmArgs {
    const void* a1;           // fp32, or FP16 when p.flags & AERO_TG_A_F16
    const void* a2;
    const void* w;            // fp32 (precision 0 / 1) or FP16 (precision 2)
    const float* bias;
    const float* addend_fn;
    const float* colscale;
    const void* residual;     // same type as out
    const float* samp_affine;
    void* out;                // fp32, or FP16 when p.flags & AERO_TG_OUT_F16
    double* stats;
    aero_tapgemm_params p;
    int ntaps;
    int tiles_t;
    int ldw;          // weight row stride (N rounded up to 4)
    int vec_a;        // 16-byte loads of A are legal
    int vec_o;        // 16-byte stores legal
    int vec_o8;       // FP16 outputs: rows are 16-byte aligned in units of 8 halves (direct lane-per-row epilogue)
    // tensor-core path: exact division of tile indices (< 2^31) by n_tiles, tiles_t, F_out:  q = (n * mul) >> shr
    uint32_t dv_mul[3], dv_shr[3];
    int direct_f16;   // FP16 outputs: same choice
    int direct_f32;   // fp32 outputs: direct lane-per-row epilogue instead of the shared-memory transpose
    int last_tile;    // tiles_total - 1 (reverse walk)
};
// tensor-core path: tile geometry and the fixed part of a CTA's shared memory, shared by the kernel and its launcher
constexpr int kBM = 128;
constexpr int kMaxStages = 8;
constexpr int kMaxBN = 128;             // widest tile of the narrow widths (32 .. 128): the whole accumulator tile is staged at once
// Wide tiles (BN = 192 / 256, FP16 operands, long K loops; tapgemm_tc.cu pick_bn): one m64n192k16 / m64n256k16 per consumer
// warpgroup and k-step.  The 96 / 128 accumulator registers per thread need setmaxnreg (producer warpgroup down to
// kProducerRegs, consumers up to kConsumerRegs), and the accumulators go through the staging tile kSliceBN columns at a time.
constexpr int kWideBN = 256;
constexpr int kSliceBN = 64;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;      // 40 * 128 + 232 * 256 = 168 * 384: the launch's register file
constexpr int kEpiWarps = 8;             // the two consumer warpgroups: two warps per 32-row quarter, alternating 16-column chunks
constexpr int kThreads = 128 + 32 * kEpiWarps;
constexpr int kATileBytes = kBM * 128;   // 16 KB

struct TcShared {
    uint64_t full[kMaxStages];
    uint64_t empty[kMaxStages];
    float stats[kEpiWarps][8][2];   // [epilogue warp][group slot][sum, sumsq]: fixed-order reduction, run-to-run deterministic
    float part[kEpiWarps][4][2];    // per-warp scratch for the fixed-order flush of the coalesced epilogue
    alignas(16) float stage[kEpiWarps][32][20];   // per-warp transpose buffer (16 columns): lane-per-row -> row-contiguous stores
};

// a tensor-core tap-GEMM kernel: (A1 map, A2 map, W map, args, stages, n-tiles, tiles)
using KernelFn = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, TapGemmArgs, int, int, int);
int tapgemm_simt_launch(const TapGemmArgs& g, cudaStream_t st);
int tapgemm_tc_launch(const TapGemmArgs& g, cudaStream_t st);
bool tapgemm_tc_eligible(const aero_tapgemm_params& p);
}  // namespace aero
