// Minimal stand-alone runner of the hot path with the reference CLI's shape:
//   b200_pipeline <pipeline> baseband <input> <output_hint> --samplerate 6e6 --baseband_format cs16 [--fused] [--key value ...]
// (cf. `satdump pipeline metop_ahrpt baseband in.cs16 out --samplerate 6e6 --baseband_format cs16`, README.md:52).
// Pipelines known here carry the module parameters of resources/pipelines/{MetOp,JPSS}.json.
#include "stream_modules.hpp"
#include <cstdio>
#include <cstring>
using namespace b200host;

// the module stats of the HRPT and Aqua DB decoders (module_noaa_hrpt_decoder.cpp:47-52, module_meteor_hrpt_decoder.cpp:52-60,
// module_aqua_db_decoder.cpp:83-93); frames: output units
static void print_hrpt_stats(const std::string &dec, long frames, int state)
{
    // module_noaa_gac_decoder.cpp:144-150 (the HRPT module's divisor, as the module has it), module_dmsp_rtd_decoder.cpp:76-82
    if (dec == "noaa_gac_decoder")
        printf("frame_count %ld\n", frames / 11090);
    if (dec == "dmsp_rtd_decoder")
        printf("deframer_state %s\n", state == 0 ? "NOSYNC" : (state == 2 ? "SYNCING" : "SYNCED"));
    if (dec == "meteor_xband_decoder")
        printf("frame_count %ld\n", frames);
    if (dec == "aqua_db_decoder")
        printf("deframer_state %s\n", state == 2 ? "NOSYNC" : (state == 6 ? "SYNCING" : "SYNCED"));
    if (dec == "fengyun_ahrpt_decoder") // module_fengyun_ahrpt_decoder.cpp:138-152: states 2 / 8 / 16
        printf("deframer_lock %d\ndeframer_state %s\n", state == 16, state == 2 ? "NOSYNC" : (state == 8 ? "SYNCING" : "SYNCED"));
    if (dec == "fengyun_mpt_decoder") // module_fengyun_mpt_decoder.cpp:137-153: states 2 / 6 / 12
        printf("deframer_lock %d\ndeframer_state %s\n", state == 12, state == 2 ? "NOSYNC" : (state == 6 ? "SYNCING" : "SYNCED"));
    if (dec == "noaa_hrpt_decoder")
        printf("frame_count %ld\n", frames / 11090);
    if (dec == "meteor_hrpt_decoder")
        printf("deframer_lock %d\ndeframer_state %s\nframe_count %ld\n", state == 12, state == 0 ? "NOSYNC" : (state == 2 || state == 6 ? "SYNCING" : "SYNCED"),
               frames);
}

int main(int argc, char **argv)
{
    if (argc < 5) {
        fprintf(stderr, "usage: %s <metop_ahrpt|jpss_hrd|npp_hrd|simple_bpsk|simple_qpsk|pm_bpsk|ldpc_qpsk|landsat|turbo_pm|turbo_bpsk|metop_dump|meteor_lrpt|noaa_hrpt|meteor_hrpt|noaa_gac|dmsp_rtd|meteor_mtvza|meteor_kmss_bpsk|fengyun_ahrpt|fengyun_ahrpt_d|fengyun_mpt|aqua_db|aura_db|terra_db|bluewalker3_wide|bluewalker3_narrow> baseband <input> <output_hint> [--fused] [--key value ...]\n", argv[0]);
        return 2;
    }
    const std::string pipe = argv[1], level = argv[2], in = argv[3], out = argv[4];
    Params dp, fp;
    std::string dec;
    if (pipe == "metop_ahrpt") { // resources/pipelines/MetOp.json:30-47
        dp = Params{{"constellation", "qpsk"}, {"symbolrate", "2333333"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.003"}};
        fp = Params{{"viterbi_outsync_after", "10"}, {"viterbi_ber_thresold", "0.28"}};
        dec = "metop_ahrpt_decoder";
    } else if (pipe == "metop_dump") { // resources/pipelines/MetOp.json "metop_dump": 35 Msym/s QPSK recorded at 45 MS/s
        dp = Params{{"constellation", "qpsk"}, {"symbolrate", "35000000"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.03"}};
        dec = "metop_dump_decoder";
    } else if (pipe == "meteor_lrpt") { // resources/pipelines/Meteor-M.json "METEOR M2 LRPT 72k": QPSK at 72 ksym/s, 1 MS/s by default
        dp = Params{{"constellation", "qpsk"}, {"symbolrate", "72000"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.002"}};
        fp = Params{{"diff_decode", "false"}};
        dec = "meteor_lrpt_decoder";
    } else if (pipe == "noaa_gac" || pipe == "dmsp_rtd") { // resources/pipelines/NOAA.json "noaa_gac", DMSP.json "dmsp_rtd": psk_demod BPSK
        if (pipe == "noaa_gac") {
            dp = Params{{"constellation", "bpsk"}, {"symbolrate", "2661600"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.004"}, {"post_costas_dc", "true"}};
            fp = Params{{"backward", "false"}};
            dec = "noaa_gac_decoder";
        } else {
            dp = Params{{"constellation", "bpsk"}, {"symbolrate", "1024000"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.005"}};
            dec = "dmsp_rtd_decoder";
        }
    } else if (pipe == "meteor_mtvza" || pipe == "meteor_kmss_bpsk") { // resources/pipelines/Meteor-M.json "meteor_m_mtvza_dump",
        // "meteor_m_kmss_bpsk_db": psk_demod BPSK at 15.36 | 61.44 Msym/s (rrc_alpha 0.6, pll_bw 0.004, rrc_taps 31); the pipelines name no
        // samplerate: it comes from the command line
        const bool kmss = pipe == "meteor_kmss_bpsk";
        dp = Params{{"constellation", "bpsk"}, {"symbolrate", kmss ? "61440000" : "15360000"}, {"rrc_alpha", "0.6"}, {"pll_bw", "0.004"},
                    {"rrc_taps", "31"}};
        fp = Params{{"instrument_type", kmss ? "kmss_bpsk" : "mtvza"}};
        dec = "meteor_xband_decoder";
    } else if (pipe == "fengyun_ahrpt" || pipe == "fengyun_ahrpt_d") { // resources/pipelines/FengYun-3.json "FengYun-3 A/B AHRPT": psk_demod
        // QPSK at 2.8 Msym/s (rrc_alpha 0.5, pll_bw 0.003), and the shape of the D / E / F / G / H pipelines, which set
        // invert_second_viterbi (their symbol rates and loop settings come from the command line)
        dp = Params{{"constellation", "qpsk"}, {"symbolrate", "2800000"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.003"}};
        fp = Params{{"viterbi_outsync_after", "20"}, {"viterbi_ber_thresold", "0.26"},
                    {"invert_second_viterbi", pipe == "fengyun_ahrpt_d" ? "true" : "false"}};
        dec = "fengyun_ahrpt_decoder";
    } else if (pipe == "fengyun_mpt") { // resources/pipelines/FengYun-3.json "FengYun-3 A/B/C MPT" (fengyun3_abc_mpt): psk_demod QPSK at
        // 18.7 Msym/s (rrc_alpha 0.5, pll_bw 0.0063, costas_max_offset 1 MHz); the pipeline names no samplerate: it comes from the command line
        dp = Params{{"constellation", "qpsk"}, {"symbolrate", "18700000"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.0063"},
                    {"costas_max_offset", "1000000"}};
        fp = Params{{"viterbi_outsync_after", "20"}, {"viterbi_ber_thresold", "0.300"}};
        dec = "fengyun_mpt_decoder";
    } else if (pipe == "noaa_hrpt" || pipe == "meteor_hrpt") { // resources/pipelines/NOAA.json "noaa_hrpt", Meteor-M.json "meteor_hrpt":
        // pm_demod at 665 400 sym/s (pll_bw 0.01, rrc_alpha 0.6 | 0.5, clock_omega_relative_limit 0.001), 3 MS/s by default
        const bool noaa = pipe == "noaa_hrpt";
        dp = Params{{"b200_demod_module", "pm_demod"}, {"symbolrate", "665400"}, {"pll_bw", "0.01"}, {"rrc_alpha", noaa ? "0.6" : "0.5"},
                    {"clock_omega_relative_limit", "0.001"}};
        if (noaa)
            fp = Params{{"deframer_thresold", "10"}};
        dec = noaa ? "noaa_hrpt_decoder" : "meteor_hrpt_decoder";
    } else if (pipe == "aqua_db" || pipe == "aura_db") { // resources/pipelines/EOS.json "aqua_db", "aura_db": OQPSK at 7.5 Msym/s, 15 MS/s
        dp = Params{{"constellation", "oqpsk"}, {"symbolrate", "7500000"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.006"}, {"clock_gain_omega", "0.8"},
                    {"clock_mu", "0.9"}, {"clock_gain_mu", "0.037"}, {"clock_omega_relative_limit", "0.0001"}, {"costas_max_offset", "1e6"}};
        dec = "aqua_db_decoder";
    } else if (pipe == "terra_db") { // resources/pipelines/EOS.json "terra_db": terra_db_demod at 13.125 Msym/s, 45 MS/s, then
        // ccsds_conv_concat_decoder (bpsk_90, NRZ-M, RS I=4, the derandomiser after RS from byte 10)
        dp = Params{{"b200_demod_module", "terra_db_demod"}, {"symbolrate", "13125000"}};
        fp = Params{{"constellation", "bpsk_90"}, {"cadu_size", "8192"}, {"viterbi_ber_thresold", "0.300"}, {"viterbi_outsync_after", "20"},
                    {"derandomize", "true"}, {"derand_after_rs", "true"}, {"derand_start", "10"}, {"nrzm", "true"}, {"rs_i", "4"}, {"rs_type", "rs223"}};
        dec = "ccsds_conv_concat_decoder";
    } else if (pipe == "bluewalker3_wide" || pipe == "bluewalker3_narrow") { // resources/pipelines/BlueWalker3.json: fsk_demod at 512 | 128
        // ksym/s (rrc_alpha 0.35), then ccsds_conv_concat_decoder (bpsk_90, CADUs of 9784 | 2648 bits, derandomised, no RS). The pipeline
        // names no samplerate: it comes from the command line
        const bool wide = pipe == "bluewalker3_wide";
        dp = Params{{"b200_demod_module", "fsk_demod"}, {"symbolrate", wide ? "512000" : "128000"}, {"rrc_alpha", "0.35"}};
        fp = Params{{"constellation", "bpsk_90"}, {"cadu_size", wide ? "9784" : "2648"}, {"viterbi_ber_thresold", "0.300"}, {"viterbi_outsync_after", "20"},
                    {"derandomize", "true"}, {"rs_i", "0"}};
        dec = "ccsds_conv_concat_decoder";
    } else if (pipe == "jpss_hrd" || pipe == "npp_hrd") { // resources/pipelines/JPSS.json
        dp = Params{{"constellation", "oqpsk"}, {"symbolrate", pipe == "jpss_hrd" ? "25000000" : "15000000"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.002"}};
        fp = Params{{"constellation", "oqpsk"}, {"cadu_size", "10232"}, {"viterbi_ber_thresold", "0.3"}, {"viterbi_outsync_after", "20"},
                    {"derandomize", "true"}, {"nrzm", "true"}, {"rs_i", "5"}, {"rs_type", "rs223"}, {"rs_usecheck", "true"}};
        dec = "ccsds_conv_concat_decoder";
    } else if (pipe == "simple_bpsk" || pipe == "simple_qpsk") { // psk_demod -> ccsds_simple_psk_decoder (no convolutional code), the shape of
        // 50 shipped pipelines (e.g. resources/pipelines/FengYun-3.json:630-639); symbolrate etc. come from the command line
        const char *con = pipe == "simple_bpsk" ? "bpsk" : "qpsk";
        dp = Params{{"constellation", con}, {"symbolrate", "1200000"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.003"}};
        fp = Params{{"constellation", con}, {"cadu_size", "8192"}, {"nrzm", pipe == "simple_bpsk" ? "true" : "false"}, {"derandomize", "true"}, {"rs_i", "4"},
                    {"rs_type", "rs223"}};
        dec = "ccsds_simple_psk_decoder";
    } else if (pipe == "pm_bpsk") { // pm_demod -> ccsds_conv_concat_decoder, the shape of 14 shipped pipelines (residual-carrier PM with a BPSK
        // subcarrier; symbolrate etc. come from the command line)
        dp = Params{{"b200_demod_module", "pm_demod"}, {"symbolrate", "500000"}, {"rrc_alpha", "0.5"}, {"pll_bw", "0.01"}, {"pll_max_offset", "3.14"},
                    {"costas_bw", "0.005"}};
        fp = Params{{"constellation", "bpsk"}, {"cadu_size", "8192"}, {"viterbi_ber_thresold", "0.3"}, {"viterbi_outsync_after", "20"}, {"derandomize", "true"},
                    {"rs_i", "4"}, {"rs_type", "rs223"}};
        dec = "ccsds_conv_concat_decoder";
    } else if (pipe == "ldpc_qpsk" || pipe == "landsat") { // psk_demod -> ccsds_ldpc_decoder, rate 7/8: FengYun-3 MERSI / GOES-R raw data
        // (FengYun-3.json:530-548, GOES.json:532-560) and LandSat 8/9 with its inner stream (LandSat.json:35-63); rates from the command line
        const bool ls = pipe == "landsat";
        dp = Params{{"constellation", ls ? "oqpsk" : "qpsk"}, {"symbolrate", ls ? "2000000" : "3000000"}, {"rrc_alpha", ls ? "0.5" : "0.35"},
                    {"pll_bw", ls ? "0.002" : "0.003"}};
        fp = Params{{"constellation", ls ? "oqpsk" : "qpsk"}, {"ldpc_rate", "7/8"}, {"ldpc_iterations", "10"}, {"derandomize", "true"}};
        if (ls) {
            fp.set("internal_stream", "true");
            fp.set("internal_cadu_size", "8272");
            fp.set("internal_asm", "352EF853");
        }
        dec = "ccsds_ldpc_decoder";
    } else if (pipe == "turbo_pm") { // pm_demod -> ccsds_turbo_decoder, rate 1/2, base 1115: the shape of the Juice, TGO, ORX, Hera, Escapade
        // and Chandrayaan-3 pipelines (residual-carrier PM), with Juice's parameters (resources/pipelines/Juice.json)
        dp = Params{{"b200_demod_module", "pm_demod"}, {"symbolrate", "526316"}, {"rrc_alpha", "0.35"}, {"pll_bw", "0.002"}, {"pll_max_offset", "3.14"},
                    {"costas_bw", "0.001"}};
        fp = Params{{"turbo_rate", "1/2"}, {"turbo_base", "1115"}, {"turbo_iters", "5"}};
        dec = "ccsds_turbo_decoder";
    } else if (pipe == "turbo_bpsk") { // psk_demod BPSK -> ccsds_turbo_decoder, rate 1/6, base 1115: the shape of the Psyche and STEREO
        // pipelines, with Psyche's parameters (resources/pipelines/Psyche.json)
        dp = Params{{"constellation", "bpsk"}, {"symbolrate", "368000"}, {"rrc_alpha", "0.35"}, {"pll_bw", "0.002"}, {"post_costas_dc", "true"}};
        fp = Params{{"turbo_rate", "1/6"}, {"turbo_base", "1115"}, {"turbo_iters", "1"}};
        dec = "ccsds_turbo_decoder";
    } else {
        fprintf(stderr, "unknown pipeline %s\n", pipe.c_str());
        return 2;
    }
    bool fused = false;
    for (int i = 5; i < argc; i++) {
        if (!strcmp(argv[i], "--fused")) { fused = true; continue; }
        if (!strncmp(argv[i], "--", 2) && i + 1 < argc) { dp.set(argv[i] + 2, argv[i + 1]); fp.set(argv[i] + 2, argv[i + 1]); i++; }
    }
    if (level != "baseband") {
        fprintf(stderr, "only the 'baseband' input level is part of the hot path\n");
        return 2;
    }
    try {
        if (fused) {
            FusedStage m(dec, in, out, dp, fp);
            m.process();
            printf("wrote %s (%ld frames)\n", m.getOutput().c_str(), m.frames_written.load());
            if (dec == "metop_dump_decoder" || dec == "meteor_lrpt_decoder")
                printf("lock_state %s\n", m.correlator_lock.load() ? "SYNCED" : "NOSYNC");
            print_hrpt_stats(dec, m.frames_written.load(), m.deframer_state.load());
        } else {
            PskDemodStage m1(in, out, dp, dp.str("b200_demod_module", "psk_demod"));
            FecStage m2(dec, "", out, fp);
            run_two_stage(m1, m2);
            printf("wrote %s (%ld frames)\n", m2.getOutput().c_str(), m2.frames_written.load());
            if (dec == "metop_dump_decoder" || dec == "meteor_lrpt_decoder")
                printf("lock_state %s\n", m2.correlator_lock.load() ? "SYNCED" : "NOSYNC");
            print_hrpt_stats(dec, m2.frames_written.load(), m2.deframer_state.load());
        }
    } catch (const std::exception &e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    return 0;
}
