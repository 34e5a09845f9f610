// aero_tapgemm_fwd: validation + dispatch (fp32 SIMT tiles, or TF32 wgmma tiles when eligible).
#include "tapgemm.cuh"


extern "C" int aero_tapgemm_fwd(const void* a1, const void* a2, const void* w, const float* bias,
                                const float* addend_fn, const float* colscale, const void* residual,
                                const float* samp_affine, void* out, double* stats,
                                const aero_tapgemm_params* pp, aero_stream_t stream) {
    using namespace aero;
    AERO_REQUIRE(w && out && pp, "aero_tapgemm_fwd: null argument");
    const aero_tapgemm_params& p = *pp;
    AERO_REQUIRE(p.B >= 1 && p.F_out >= 1 && p.T >= 1 && p.N >= 1 && p.F_in >= 1 && p.T_in >= 1, "aero_tapgemm_fwd: bad sizes");
    AERO_REQUIRE(p.C1 >= 0 && p.C2 >= 0 && p.C1 + p.C2 >= 1, "aero_tapgemm_fwd: C1=%d C2=%d", p.C1, p.C2);
    AERO_REQUIRE((p.C1 == 0 || a1) && (p.C2 == 0 || a2), "aero_tapgemm_fwd: missing source pointer");
    AERO_REQUIRE(p.kf >= 1 && p.kt >= 1 && p.stride_f >= 1, "aero_tapgemm_fwd: taps");
    int ntaps;
    if (p.mode == AERO_TAPS_CONV) {
        ntaps = p.kf * p.kt;
    } else if (p.mode == AERO_TAPS_CONVT) {
        AERO_REQUIRE(p.kt == 1 && p.kf % p.stride_f == 0, "aero_tapgemm_fwd: transposed conv needs kt=1 and kf %% stride == 0");
        ntaps = p.kf / p.stride_f;
    } else if (p.mode == AERO_TAPS_MIX) {
        AERO_REQUIRE(p.precision == 1 || p.precision == 2, "aero_tapgemm_fwd: AERO_TAPS_MIX exists on the wgmma path only (precision 1 / 2)");
        ntaps = 1;
    } else {
        set_error("aero_tapgemm_fwd: mode=%d", p.mode);
        return AERO_ERR_INVALID;
    }
    AERO_REQUIRE(p.act >= AERO_ACT_NONE && p.act <= AERO_ACT_TANH, "aero_tapgemm_fwd: act=%d", p.act);
    AERO_REQUIRE(!p.glu || p.N % 2 == 0, "aero_tapgemm_fwd: GLU needs even N");
    const int Nout = p.glu ? p.N / 2 : p.N;
    if (p.stats_mode) {
        AERO_REQUIRE(stats, "aero_tapgemm_fwd: stats buffer missing");
        AERO_REQUIRE(p.stats_mode == 1 || p.stats_mode == 2, "aero_tapgemm_fwd: stats_mode");
        if (p.stats_mode == 1) {
            AERO_REQUIRE(p.groups >= 1 && Nout % p.groups == 0, "aero_tapgemm_fwd: groups");
            const int gw = Nout / p.groups;
            const int tno = p.N <= 16 ? 1 : (p.glu ? 2 : 4);       // output columns per thread
            const int tile_w = p.N <= 16 ? 16 : (p.glu ? 32 : 64);  // output columns per CTA
            AERO_REQUIRE(gw % tno == 0 && tile_w / gw + 2 <= 8,
                         "aero_tapgemm_fwd: group width %d not supported by the statistics epilogue", gw);
        }
    }
    AERO_REQUIRE(!(p.glu && p.N <= 16), "aero_tapgemm_fwd: GLU with N <= 16 unsupported");
    TapGemmArgs g;
    g.a1 = a1; g.a2 = a2; g.w = w; g.bias = bias; g.addend_fn = addend_fn; g.colscale = colscale;
    g.residual = residual; g.samp_affine = samp_affine; g.out = out; g.stats = stats;
    g.p = p; g.ntaps = ntaps; g.tiles_t = 0;
    g.ldw = (p.N + 3) & ~3;
    auto al16 = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
    g.vec_a = (p.C1 % 4 == 0) && (p.C2 % 4 == 0) &&
              (p.C1 == 0 || (al16(a1) && p.a1_sb % 4 == 0 && p.a1_sf % 4 == 0 && p.a1_st % 4 == 0)) &&
              (p.C2 == 0 || (al16(a2) && p.a2_sb % 4 == 0 && p.a2_sf % 4 == 0 && p.a2_st % 4 == 0));
    g.vec_o = al16(out) && p.o_sb % 4 == 0 && p.o_sf % 4 == 0 && p.o_st % 4 == 0 && Nout % 4 == 0 &&
              (!residual || (al16(residual) && p.r_sb % 4 == 0 && p.r_sf % 4 == 0 && p.r_st % 4 == 0)) &&
              (!addend_fn || al16(addend_fn));
    g.vec_o8 = g.vec_o && p.o_sb % 8 == 0 && p.o_sf % 8 == 0 && p.o_st % 8 == 0 && Nout % 8 == 0 &&
               (!residual || (p.r_sb % 8 == 0 && p.r_sf % 8 == 0 && p.r_st % 8 == 0));
    AERO_REQUIRE(al16(w) && p.w_sb % 4 == 0, "aero_tapgemm_fwd: weights must be 16-byte aligned");
    AERO_REQUIRE(p.precision >= 0 && p.precision <= 2, "aero_tapgemm_fwd: precision=%d", p.precision);
    AERO_REQUIRE((p.precision != 1 || !(p.flags & AERO_TG_A_F16)) && (p.precision != 2 || (p.flags & AERO_TG_A_F16)),
                 "aero_tapgemm_fwd: precision 1 reads fp32 sources, precision 2 FP16 sources (flags=%d)", p.flags);
    if (p.precision >= 1) {
        if (!tapgemm_tc_eligible(p)) {
            set_error("aero_tapgemm_fwd: wgmma path requested for a shape the wgmma path does not take (N=%d K=%d)", p.N, p.C1 + p.C2);
            return AERO_ERR_UNSUPPORTED;
        }
        AERO_REQUIRE((p.C1 == 0 || al16(a1)) && (p.C2 == 0 || al16(a2)), "aero_tapgemm_fwd: TMA sources must be 16-byte aligned");
        return tapgemm_tc_launch(g, (cudaStream_t)stream);
    }
    return tapgemm_simt_launch(g, (cudaStream_t)stream);
}

extern "C" int aero_tapgemm_tc_eligible(const aero_tapgemm_params* p) { return p && aero::tapgemm_tc_eligible(*p) ? 1 : 0; }
