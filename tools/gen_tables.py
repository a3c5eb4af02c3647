#!/usr/bin/env python3
"""Generate solo_b200/csrc/sb_tables_data.inc from the compiled reference libraries.

The codec's interoperability constants (entropy-coder CDFs, NLSF / LTP / high-band codebooks, QMF
prototype filter, ...) are *data* defined by the SOLO bitstream format.  They are extracted by
VALUE from the data segments of oracle/_ref/libjc1_fix.so / libjc1_flp.so (the reference compiled
by oracle/Makefile) and re-emitted in this project's own X-macro layout; no reference source text
is read or copied.  Run in the build container (needs oracle/_ref):

    make -C oracle && python tools/gen_tables.py

The generated .inc is committed so that the GPU box (no /root/reference) can build.
Each entry: (our_name, lib, symbol, element ctype, count).  Pointer tables of the reference
(NLSF CDF start pointers, LTP pointer arrays) are flattened into offset arrays.
"""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
OUT = os.path.join(ROOT, "solo_b200", "csrc", "sb_tables_data.inc")

I16, U16, I32, F32 = "i16", "u16", "i32", "f32"
CT = {I16: C.c_int16, U16: C.c_uint16, I32: C.c_int32, F32: C.c_float}

TABLES = [
    # --- QMF / high band (libBWE) ---
    ("qmf_fix", "fix", "AGR_Sate_qmf_coeffs_fix", I16, 64),
    ("qmf_flt", "flp", "AGR_Sate_qmf_coeffs", F32, 64),
    ("hb_lsp_cb1_fix", "fix", "AGR_Sate_highband_lsp_cdbk1_fix", I16, 256 * 8),
    ("hb_lsp_cb2_fix", "fix", "AGR_Sate_highband_lsp_cdbk2_fix", I16, 16 * 8),
    ("hb_gain_cb_fix", "fix", "AGR_Sate_highband_gain_cdbk_fix", I16, 32),
    ("hb_lsp_cb1_flt", "flp", "AGR_Sate_highband_lsp_cdbk1", F32, 256 * 8),
    ("hb_lsp_cb2_flt", "flp", "AGR_Sate_highband_lsp_cdbk2", F32, 16 * 8),
    ("hb_gain_cb_flt", "flp", "AGR_Sate_highband_gain_cdbk", F32, 32),
    # --- NLSF codebooks, order 10 ---
    ("nlsf_cb0_q15", "fix", "SKP_Silk_NLSF_MSVQ_CB0_10_Q15", I16, 1200),
    ("nlsf_cb0_rates_q5", "fix", "SKP_Silk_NLSF_MSVQ_CB0_10_rates_Q5", I16, 120),
    ("nlsf_cb0_ndelta_min_q15", "fix", "SKP_Silk_NLSF_MSVQ_CB0_10_ndelta_min_Q15", I32, 11),
    ("nlsf_cb0_cdf", "fix", "SKP_Silk_NLSF_MSVQ_CB0_10_CDF", U16, 126),
    ("nlsf_cb0_cdf_mid", "fix", "SKP_Silk_NLSF_MSVQ_CB0_10_CDF_middle_idx", I32, 6),
    ("nlsf_cb1_q15", "fix", "SKP_Silk_NLSF_MSVQ_CB1_10_Q15", I16, 720),
    ("nlsf_cb1_rates_q5", "fix", "SKP_Silk_NLSF_MSVQ_CB1_10_rates_Q5", I16, 72),
    ("nlsf_cb1_ndelta_min_q15", "fix", "SKP_Silk_NLSF_MSVQ_CB1_10_ndelta_min_Q15", I32, 11),
    ("nlsf_cb1_cdf", "fix", "SKP_Silk_NLSF_MSVQ_CB1_10_CDF", U16, 78),
    ("nlsf_cb1_cdf_mid", "fix", "SKP_Silk_NLSF_MSVQ_CB1_10_CDF_middle_idx", I32, 6),
    ("lsf_cos_q12", "fix", "SKP_Silk_LSFCosTab_FIX_Q12", I32, 129),
    # --- NLSF codebooks, order 16 (the 16 kHz core of 32 kHz streams) ---
    ("nlsf16_cb0_q15", "fix", "SKP_Silk_NLSF_MSVQ_CB0_16_Q15", I16, 216 * 16),
    ("nlsf16_cb0_rates_q5", "fix", "SKP_Silk_NLSF_MSVQ_CB0_16_rates_Q5", I16, 216),
    ("nlsf16_cb0_ndelta_min_q15", "fix", "SKP_Silk_NLSF_MSVQ_CB0_16_ndelta_min_Q15", I32, 17),
    ("nlsf16_cb0_cdf", "fix", "SKP_Silk_NLSF_MSVQ_CB0_16_CDF", U16, 226),
    ("nlsf16_cb0_cdf_mid", "fix", "SKP_Silk_NLSF_MSVQ_CB0_16_CDF_middle_idx", I32, 10),
    ("nlsf16_cb1_q15", "fix", "SKP_Silk_NLSF_MSVQ_CB1_16_Q15", I16, 104 * 16),
    ("nlsf16_cb1_rates_q5", "fix", "SKP_Silk_NLSF_MSVQ_CB1_16_rates_Q5", I16, 104),
    ("nlsf16_cb1_ndelta_min_q15", "fix", "SKP_Silk_NLSF_MSVQ_CB1_16_ndelta_min_Q15", I32, 17),
    ("nlsf16_cb1_cdf", "fix", "SKP_Silk_NLSF_MSVQ_CB1_16_CDF", U16, 114),
    ("nlsf16_cb1_cdf_mid", "fix", "SKP_Silk_NLSF_MSVQ_CB1_16_CDF_middle_idx", I32, 10),
    ("nlsf_interp_cdf", "fix", "SKP_Silk_NLSF_interpolation_factor_CDF", U16, 6),
    ("nlsf_interp_offset", "fix", "SKP_Silk_NLSF_interpolation_factor_offset", I32, 1),
    # --- LTP ---
    ("ltp_vq0_q14", "fix", "SKP_Silk_LTP_gain_vq_0_Q14", I16, 50),
    ("ltp_vq1_q14", "fix", "SKP_Silk_LTP_gain_vq_1_Q14", I16, 100),
    ("ltp_vq2_q14", "fix", "SKP_Silk_LTP_gain_vq_2_Q14", I16, 200),
    ("ltp_bits0_q6", "fix", "SKP_Silk_LTP_gain_BITS_Q6_0", I16, 10),
    ("ltp_bits1_q6", "fix", "SKP_Silk_LTP_gain_BITS_Q6_1", I16, 20),
    ("ltp_bits2_q6", "fix", "SKP_Silk_LTP_gain_BITS_Q6_2", I16, 40),
    ("ltp_cdf0", "fix", "SKP_Silk_LTP_gain_CDF_0", U16, 11),
    ("ltp_cdf1", "fix", "SKP_Silk_LTP_gain_CDF_1", U16, 21),
    ("ltp_cdf2", "fix", "SKP_Silk_LTP_gain_CDF_2", U16, 41),
    ("ltp_cdf_offsets", "fix", "SKP_Silk_LTP_gain_CDF_offsets", I32, 3),
    ("ltp_vq_sizes", "fix", "SKP_Silk_LTP_vq_sizes", I32, 3),
    ("ltp_mid_avg_rd_q14", "fix", "SKP_Silk_LTP_gain_middle_avg_RD_Q14", I32, 1),
    ("ltp_per_index_cdf", "fix", "SKP_Silk_LTP_per_index_CDF", U16, 4),
    ("ltp_per_index_offset", "fix", "SKP_Silk_LTP_per_index_CDF_offset", I32, 1),
    ("ltpscale_cdf", "fix", "SKP_Silk_LTPscale_CDF", U16, 4),
    ("ltpscale_offset", "fix", "SKP_Silk_LTPscale_offset", I32, 1),
    ("ltpscales_q14", "fix", "SKP_Silk_LTPScales_table_Q14", I16, 3),
    ("ltpscale_thresholds_q15", "fix", "LTPScaleThresholds_Q15", I16, 11),
    # --- pitch ---
    ("pitch_cb_lags_stage2", "fix", "SKP_Silk_CB_lags_stage2", I16, 44),
    ("pitch_lag_nb_cdf", "fix", "SKP_Silk_pitch_lag_NB_CDF", U16, 130),
    ("pitch_lag_nb_offset", "fix", "SKP_Silk_pitch_lag_NB_CDF_offset", I32, 1),
    ("pitch_contour_nb_cdf", "fix", "SKP_Silk_pitch_contour_NB_CDF", U16, 12),
    ("pitch_contour_nb_offset", "fix", "SKP_Silk_pitch_contour_NB_CDF_offset", I32, 1),
    ("pitch_lag_wb_cdf", "fix", "SKP_Silk_pitch_lag_WB_CDF", U16, 258),
    ("pitch_lag_wb_offset", "fix", "SKP_Silk_pitch_lag_WB_CDF_offset", I32, 1),
    ("pitch_contour_cdf", "fix", "SKP_Silk_pitch_contour_CDF", U16, 35),
    ("pitch_contour_offset", "fix", "SKP_Silk_pitch_contour_CDF_offset", I32, 1),
    ("pitch_cb_lags_stage3", "fix", "SKP_Silk_CB_lags_stage3", I16, 4 * 34),
    # --- gains ---
    ("gain_cdf", "fix", "SKP_Silk_gain_CDF", U16, 130),
    ("gain_cdf_offset", "fix", "SKP_Silk_gain_CDF_offset", I32, 1),
    ("delta_gain_cdf", "fix", "SKP_Silk_delta_gain_CDF", U16, 46),
    ("delta_gain_cdf_offset", "fix", "SKP_Silk_delta_gain_CDF_offset", I32, 1),
    ("md_delta_gain_cdf", "fix", "SKP_Silk_md_delta_gain_CDF", U16, 9),
    ("md_delta_gain_cdf_offset", "fix", "SKP_Silk_md_delta_gain_CDF_offset", I32, 1),
    # --- misc side info ---
    ("type_offset_cdf", "fix", "SKP_Silk_type_offset_CDF", U16, 5),
    ("type_offset_cdf_offset", "fix", "SKP_Silk_type_offset_CDF_offset", I32, 1),
    ("type_offset_joint_cdf", "fix", "SKP_Silk_type_offset_joint_CDF", U16, 20),
    ("sampling_rates_cdf", "fix", "SKP_Silk_SamplingRates_CDF", U16, 5),
    ("sampling_rates_offset", "fix", "SKP_Silk_SamplingRates_offset", I32, 1),
    ("sampling_rates_table", "fix", "SKP_Silk_SamplingRates_table", I32, 4),
    ("seed_cdf", "fix", "SKP_Silk_Seed_CDF", U16, 5),
    ("seed_offset", "fix", "SKP_Silk_Seed_offset", I32, 1),
    ("vadflag_cdf", "fix", "SKP_Silk_vadflag_CDF", U16, 3),
    ("vadflag_offset", "fix", "SKP_Silk_vadflag_offset", I32, 1),
    ("frame_term_cdf", "fix", "SKP_Silk_FrameTermination_CDF", U16, 5),
    ("frame_term_offset", "fix", "SKP_Silk_FrameTermination_offset", I32, 1),
    ("md_index_cdf", "fix", "SKP_Silk_writeMDIndex_CDF", U16, 3),
    ("md_index_offset", "fix", "SKP_Silk_writeMDIndex_offset", I32, 1),
    ("lsb_cdf", "fix", "SKP_Silk_lsb_CDF", U16, 3),
    # --- pulses ---
    ("max_pulses_table", "fix", "SKP_Silk_max_pulses_table", I32, 4),
    ("pulses_per_block_cdf", "fix", "SKP_Silk_pulses_per_block_CDF", U16, 210),
    ("pulses_per_block_cdf_offset", "fix", "SKP_Silk_pulses_per_block_CDF_offset", I32, 1),
    ("pulses_per_block_bits_q6", "fix", "SKP_Silk_pulses_per_block_BITS_Q6", I16, 180),
    ("rate_levels_cdf", "fix", "SKP_Silk_rate_levels_CDF", U16, 20),
    ("rate_levels_cdf_offset", "fix", "SKP_Silk_rate_levels_CDF_offset", I32, 1),
    ("rate_levels_bits_q6", "fix", "SKP_Silk_rate_levels_BITS_Q6", I16, 18),
    ("shell_table0", "fix", "SKP_Silk_shell_code_table0", U16, 33),
    ("shell_table1", "fix", "SKP_Silk_shell_code_table1", U16, 52),
    ("shell_table2", "fix", "SKP_Silk_shell_code_table2", U16, 102),
    ("shell_table3", "fix", "SKP_Silk_shell_code_table3", U16, 207),
    ("shell_table_offsets", "fix", "SKP_Silk_shell_code_table_offsets", U16, 19),
    ("sign_cdf", "fix", "SKP_Silk_sign_CDF", U16, 36),
    ("quant_offsets_q10", "fix", "SKP_Silk_Quantization_Offsets_Q10", I16, 4),
    # --- rate control / misc ---
    ("snr_table_q1", "fix", "SNR_table_Q1", I32, 8),
    ("target_rate_table_nb", "fix", "TargetRate_table_NB", I32, 8),
    ("resampler_down2_0", "fix", "SKP_Silk_resampler_down2_0", I16, 1),
    ("resampler_down2_1", "fix", "SKP_Silk_resampler_down2_1", I16, 1),
    ("sine_freq_table_q16", "fix", "freq_table_Q16", I16, 27),
]

# pointer tables of the reference flattened to element offsets: (our_name, lib, ptr_symbol, n, base_symbol, elem_size)
PTR_TABLES = [
    ("nlsf_cb0_cdf_start", "fix", "SKP_Silk_NLSF_MSVQ_CB0_10_CDF_start_ptr", 6, "SKP_Silk_NLSF_MSVQ_CB0_10_CDF", 2),
    ("nlsf_cb1_cdf_start", "fix", "SKP_Silk_NLSF_MSVQ_CB1_10_CDF_start_ptr", 6, "SKP_Silk_NLSF_MSVQ_CB1_10_CDF", 2),
    ("nlsf16_cb0_cdf_start", "fix", "SKP_Silk_NLSF_MSVQ_CB0_16_CDF_start_ptr", 10, "SKP_Silk_NLSF_MSVQ_CB0_16_CDF", 2),
    ("nlsf16_cb1_cdf_start", "fix", "SKP_Silk_NLSF_MSVQ_CB1_16_CDF_start_ptr", 10, "SKP_Silk_NLSF_MSVQ_CB1_16_CDF", 2),
]


def symtab(path):
    out = subprocess.check_output(["nm", "-S", "--defined-only", path], text=True)
    tab = {}
    for line in out.splitlines():
        p = line.split()
        if len(p) == 4:
            tab[p[3]] = (int(p[0], 16), int(p[1], 16))
    return tab


class Lib:
    def __init__(self, kind):
        path = os.path.join(REF, "libjc1_%s.so" % kind)
        self.lib = C.CDLL(path)
        self.tab = symtab(path)
        # load bias from one exported function
        anchor = "AGR_Sate_Encoder_Init"
        addr = C.cast(getattr(self.lib, anchor), C.c_void_p).value
        self.bias = addr - self.tab[anchor][0]

    def read(self, sym, ctype, n):
        off, size = self.tab[sym]
        assert size == C.sizeof(ctype) * n, "%s: size %d != %d*%d" % (sym, size, C.sizeof(ctype), n)
        return list((ctype * n).from_address(self.bias + off))

    def addr(self, sym):
        return self.bias + self.tab[sym][0]


def fmt(v, t):
    if t == F32:
        s = "%.9g" % v  # 9 significant digits round-trip an IEEE binary32 exactly
        if "." not in s and "e" not in s and "n" not in s:
            s += ".0"
        return s + "f"
    return str(int(v))


def main():
    libs = {"fix": Lib("fix"), "flp": Lib("flp")}
    lines = [
        "// GENERATED by tools/gen_tables.py from the data segments of oracle/_ref/libjc1_{fix,flp}.so -- do not edit.",
        "// Bitstream-format constants of the SOLO codec (values only), X-macro layout: SB_TAB(type, name, count, values...)",
        "",
    ]
    for name, kind, sym, t, n in TABLES:
        vals = libs[kind].read(sym, CT[t], n)
        body = ",".join(fmt(v, t) for v in vals)
        lines.append("SB_TAB(%s, %s, %d, %s)" % (t, name, n, body))
    for name, kind, psym, n, bsym, esz in PTR_TABLES:
        L = libs[kind]
        ptrs = L.read(psym, C.c_uint64, n)
        base = L.addr(bsym)
        offs = [(p - base) // esz for p in ptrs]
        lines.append("SB_TAB(i32, %s, %d, %s)" % (name, n, ",".join(map(str, offs))))
    # NLSF stage sizes (from the Stage_info structs: nVectors is the first int32 of each 24-byte entry)
    for order, prefix in ((10, "nlsf"), (16, "nlsf16")):
        for cb in (0, 1):
            L = libs["fix"]
            off, size = L.tab["SKP_Silk_NLSF_CB%d_%d_Stage_info" % (cb, order)]
            raw = (C.c_uint8 * size).from_address(L.bias + off)
            nv = [int.from_bytes(bytes(raw[i * 24:i * 24 + 4]), "little") for i in range(size // 24)]
            lines.append("SB_TAB(i32, %s_cb%d_nvec, %d, %s)" % (prefix, cb, len(nv), ",".join(map(str, nv))))
    with open(OUT, "w") as f:
        f.write("\n".join(lines) + "\n")
    print("wrote", OUT, len(lines), "lines")


if __name__ == "__main__":
    sys.exit(main())
