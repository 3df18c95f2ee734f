/*
 * b200dsp — C ABI of the H100-native (sm_90a) SatDump baseband -> CADU hot path.
 *
 * This is the boundary a SatDump plugin binds (INTEGRATION.md shows the ProcessingModule shim). It
 * sits one level below SatDump's C++ plugin ABI so that the CUDA library is independent of the host
 * compiler / STL: plain pointers, sizes and POD structs only, caller-owned host buffers, opaque handles.
 *
 * Each entry point names the reference interface it replaces (paths relative to the SatDump tree):
 *
 *   b200_demod_*   the DSP chain PSKDemodModule builds and runs
 *                    src-core/pipeline/modules/demod/module_psk_demod.cpp:86-236   (init / process)
 *                    src-core/pipeline/modules/demod/module_demod_base.cpp:59-208   (initb: source, AGC)
 *                    plugins/dvb_support/dvbs2/module_dvbs2_demod.cpp:98-102        (AGC->RRC->M&M front half; constellation NONE)
 *                    src-core/pipeline/modules/demod/module_pm_demod.cpp:61-160      (PMDemodModule: cfg.pm_demod = 1)
 *                    src-core/pipeline/modules/demod/module_fsk_demod.cpp:59-158     (FSKDemodModule: cfg.fsk_demod = 1)
 *   b200_fec_*     the decoder modules
 *                    plugins/noaa_metop_support/metop/module_metop_ahrpt_decoder.cpp:34-90      (kind METOP)
 *                    src-core/pipeline/modules/ccsds/module_ccsds_conv_concat_decoder.cpp:140-200 (kind CCSDS, r=1/2)
 *                    src-core/pipeline/modules/ccsds/module_ccsds_ldpc_decoder.cpp:134-277       (kind LDPC, ldpc_rate "7/8")
 *                    src-core/pipeline/modules/ccsds/module_ccsds_turbo_decoder.cpp:137-235      (kind TURBO)
 *                    plugins/noaa_metop_support/metop/module_metop_dump_decoder.cpp:27-83        (kind METOP_DUMP)
 *                    plugins/meteor_support/meteor/module_meteor_lrpt_decoder.cpp:101-262        (kind METEOR_LRPT)
 *                    plugins/eos_support/aqua/module_aqua_db_decoder.cpp:27-83                    (kind AQUA_DB)
 *   b200_chain_*   both modules joined the way Pipeline::run joins them with a byte FIFO
 *                    src-core/pipeline/pipeline_run.cpp:44-117 — here the int8 soft stream never leaves HBM.
 *   b200_demux_*   the step behind the decoder: CADUs -> CCSDS space packets
 *                    src-core/common/ccsds/ccsds_aos/demuxer.cpp:64-199 (one Demuxer per virtual channel), vcdu.cpp:10-17, mpdu.cpp:9-13,
 *                    as plugins/noaa_metop_support/metop/module_metop_instruments.cpp:66-140 calls them
 *
 * All functions return 0 on success or a negative B200_E* code; b200_last_error() gives the text.
 * There is no CPU fallback: without a CUDA device every create() fails with B200_ENODEV.
 */
#ifndef B200DSP_H
#define B200DSP_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_EINVAL -1     /* bad / unsupported parameter (the C++ module turns this into satdump_exception) */
#define B200_ENODEV -2     /* no CUDA device / wrong architecture */
#define B200_ECUDA -3      /* CUDA runtime failure */
#define B200_ENOMEM -4
#define B200_ESTATE -5     /* e.g. pull before push, batch larger than max_batch */
#define B200_EUNSUPPORTED -6 /* option / signal condition this build does not cover (the text says which) */

/* constellation (module param "constellation", module_psk_demod.cpp:17-21; NONE = no Costas loop) */
enum { B200_BPSK = 0, B200_QPSK = 1, B200_OQPSK = 2, B200_8PSK = 3, B200_NONE = 4, B200_BPSK_90 = 5 };
/* baseband_format (common/dsp/io/baseband_type.h:7-21) */
enum { B200_CF32 = 0, B200_CS16 = 1, B200_CS8 = 2 };
/* decoder kind */
enum { B200_FEC_METOP = 0, B200_FEC_CCSDS = 1, B200_FEC_SIMPLE = 2, B200_FEC_LDPC = 3, B200_FEC_TURBO = 4, B200_FEC_METOP_DUMP = 5,
       B200_FEC_METEOR_LRPT = 6, B200_FEC_NOAA_HRPT = 7 /* noaa_hrpt_decoder */, B200_FEC_METEOR_HRPT = 8 /* meteor_hrpt_decoder */,
       B200_FEC_AQUA_DB = 9 /* aqua_db_decoder */, B200_FEC_NOAA_GAC = 10 /* noaa_gac_decoder */, B200_FEC_DMSP_RTD = 11 /* dmsp_rtd_decoder */,
       B200_FEC_METEOR_XBAND = 12 /* meteor_xband_decoder */, B200_FEC_FENGYUN_AHRPT = 13 /* fengyun_ahrpt_decoder */,
       B200_FEC_FENGYUN_MPT = 14 /* fengyun_mpt_decoder */ };
/* debug stage ids for b200_demod_debug_stage */
enum { B200_STAGE_AGC = 0, B200_STAGE_FIR = 1, B200_STAGE_COSTAS = 2, B200_STAGE_RESAMP = 3, B200_STAGE_DC = 4, B200_STAGE_MM = 5,
       B200_STAGE_PLL = 6 /* pm_demod: PLLCarrierTrackingBlock output */, B200_STAGE_PM = 7 /* pm_demod: PMToBPSK output */,
       /* fsk_demod: one float per sample; B200_STAGE_FIR and B200_STAGE_MM then give one float per sample / symbol too */
       B200_STAGE_QUAD = 8 /* QuadratureDemodBlock output */, B200_STAGE_DC2 = 9 /* CorrectIQBlock<float> output */,
       B200_STAGE_AGC2 = 10 /* AGCBlock<float> output */ };
/* mode bits of b200_demod_debug_run_stage */
#define B200_DEBUG_STRICT 1     /* the reference's operation order: separate multiply and add, left to right (generic VOLK, no FMA) */
#define B200_DEBUG_SEQUENTIAL 2 /* one segment: the feedback loop runs as ONE sequential thread from the initial state */

typedef struct b200_demod_cfg
{
    double samplerate;        /* "samplerate"  (module_demod_base.cpp:17-20)                     */
    double symbolrate;        /* "symbolrate"  (:26-27)                                          */
    int constellation;        /* "constellation"                                                 */
    float rrc_alpha;          /* "rrc_alpha"   (module_psk_demod.cpp:23-26)                      */
    int rrc_taps;             /* "rrc_taps", default 31 (module_psk_demod.h:31); only 31 built   */
    float pll_bw;             /* "pll_bw"                                                        */
    float agc_rate;           /* "agc_rate", default 1e-2 (module_demod_base.h:54)               */
    float clock_gain_omega;   /* default pow(8.7e-3,2)/4 (module_psk_demod.h:36)                 */
    float clock_mu;           /* default 0.5                                                     */
    float clock_gain_mu;      /* default 8.7e-3                                                  */
    float clock_omega_limit;  /* "clock_omega_relative_limit", default 0.005                     */
    float costas_max_offset;  /* rad/sample, default 1.0 (module_psk_demod.cpp:116-118)          */
    int format;               /* "baseband_format": B200_CF32 / CS16 / CS8                       */
    int device;               /* CUDA device ordinal                                             */
    long max_batch;           /* largest nsamples of one push (device buffers are sized for it)  */
    int keep_stages;          /* !=0: keep AGC/FIR/Costas stage outputs for b200_demod_debug_stage */
    int iq_swap;              /* "iq_swap": re <-> im at the reader (dsp/io/file_source.cpp:31-33)    */
    double final_samplerate;  /* 0 = samplerate. Otherwise the rate BaseDemodModule::initb resamples to when samplerate/symbolrate is
                                 outside [min_sps, max_sps] (module_demod_base.cpp:59-87,203-204): use b200_demod_final_samplerate().
                                 Only the rational part of SmartResamplerBlock is built: samplerate / final_samplerate must be < 2 */
    int dc_block;             /* "dc_block": CorrectIQBlock in front (utils/correct_iq.cpp:18-35, module_demod_base.cpp:113-114) */
    int post_costas_dc;       /* "post_costas_dc": CorrectIQBlock between the Costas loop and the clock recovery
                                 (module_psk_demod.cpp:127-134); not with OQPSK                                         */
    int front_resample;       /* 0: the resampler runs iff final_samplerate differs from samplerate. 2: never - BaseDemodModule::initb's
                                 `resample` is false (samplerate / symbolrate inside [min_sps, max_sps]) although "custom_samplerate" set
                                 another final_samplerate: the reference then only designs the RRC and the clock recovery for that rate
                                 (module_demod_base.cpp:66,73-74,203-204); b200_demod_resample_decision() tells                        */
    int clock_recovery;       /* 0: MMClockRecoveryBlock<complex_t> (what psk_demod builds, module_psk_demod.cpp:134-135);
                                 1: dsp::GardnerClockRecoveryBlock<complex_t> with the same arguments
                                 (common/dsp/clock_recovery/clock_recovery_gardner.cpp:33-131; SURVEY row G)                          */
    /* pm_demod (src-core/pipeline/modules/demod/module_pm_demod.cpp:12-88): AGC -> PLLCarrierTrackingBlock -> PMToBPSK ->
       [SmartResamplerBlock -> AGCBlock(0.001, 1, 1, 1000)] -> RRC -> Costas loop (order 2) -> M&M, soft = clamp(real * 100).
       The working-rate window is then [1.1, 10] samples per symbol (MAX_SPS = 10, :56) */
    int pm_demod;             /* != 0: build PMDemodModule's chain; constellation must be B200_BPSK, pll_bw above is its "costas_bw"  */
    float pm_pll_bw;          /* "pll_bw": carrier PLL loop bandwidth (required by the module, :21-24)                              */
    float pm_pll_max_offset;  /* "pll_max_offset", default 0.5 rad/sample (module_pm_demod.h:29)                                    */
    int pm_resample_after_pll;/* "resample_after_pll": the front-end resampler sits behind PMToBPSK, followed by the second AGC      */
    double pm_subcarrier_offset; /* "subcarrier_offset" Hz (uint64 in the module); 0 = the symbol rate (:67)                           */
    double freq_shift;        /* "freq_shift" Hz (long in the module): FreqShiftBlock behind the reader / DC blocker, in front of the
                                 resampler (module_demod_base.cpp:37,122-123; common/dsp/utils/freq_shift.cpp); 0 = none             */
    /* psk_demod "has_carrier" (module_psk_demod.cpp:39-40,93-116): BPSK on a residual carrier: RRC -> PLLCarrierTrackingBlock ->
       CorrectIQBlock -> Costas loop (whose frequency limit then defaults to 0.2 rad/sample: pass it in costas_max_offset) */
    int has_carrier;
    float carrier_pll_bw;         /* "carrier_pll_bw" (required by the module in this mode)   */
    float carrier_pll_max_offset; /* "carrier_pll_max_offset", default 3.14                    */
    /* fsk_demod (module_fsk_demod.cpp:13-84): the base front end and AGC -> QuadratureDemodBlock(1.0) -> CorrectIQBlock<float> ->
       AGCBlock<float>(0.1, 0.5, 1.0, 65535) -> RRC (FIRBlock<float>) -> MMClockRecoveryBlock<float>; soft = clamp(symbol * 50), one byte
       per symbol; b200_demod_pull_symbols returns one float per symbol. constellation must be B200_BPSK; pll_bw is not read. Not with
       pm_demod, has_carrier, post_costas_dc or clock_recovery 1. The module's clock defaults differ from psk_demod's: gain_omega
       pow(1.7e-2, 2) / 4, gain_mu 1.7e-2 (module_fsk_demod.h:28-31) */
    int fsk_demod;
} b200_demod_cfg;

typedef struct b200_fec_cfg
{
    int kind;                 /* B200_FEC_METOP (metop_ahrpt_decoder) | B200_FEC_CCSDS (ccsds_conv_concat_decoder) |
                                 B200_FEC_SIMPLE (ccsds_simple_psk_decoder: no convolutional code,
                                 src-core/pipeline/modules/ccsds/module_ccsds_simple_psk_decoder.cpp)                */
    int constellation;        /* ccsds: B200_BPSK / BPSK_90 / QPSK / OQPSK; simple: B200_BPSK / QPSK */
    int cadu_size;            /* bits ("cadu_size"); METOP: 8192                                 */
    int outsync_after;        /* "viterbi_outsync_after"                                         */
    float ber_thresold;       /* "viterbi_ber_thresold"                                          */
    int nrzm, derandomize, derand_after_rs, derand_start;
    int rs_i, rs_dualbasis, rs_fill_bytes, rs_usecheck, rs_type;
    int iq_invert;
    unsigned int asm_sync;    /* "asm", default 0x1ACFFC1D                                       */
    int device;
    long max_soft;            /* largest number of soft bytes of one push                        */
    int qpsk_swap_iq;         /* simple: "qpsk_swap_iq"   (module_ccsds_simple_psk_decoder.cpp:27)    */
    int qpsk_swap_diff;       /* simple: "qpsk_swap_diff", default true (:28); used with nrzm on QPSK  */
    int oqpsk_delay;          /* simple: "oqpsk_delay" (:29)                                          */
    int conv_rate;            /* ccsds: "conv_rate" (module_ccsds_conv_concat_decoder.cpp:33,99-117): 0 = "1/2" (Viterbi1_2); 2, 3, 5, 7 = "2/3",
                                 "3/4", "5/6", "7/8" (Viterbi_Depunc, common/codings/viterbi/viterbi_punc.cpp + depunc.h)           */
    /* kind B200_FEC_LDPC = ccsds_ldpc_decoder (module_ccsds_ldpc_decoder.cpp:19-124): correlator on the 32-bit ASM 0x1ACFFC1D over
       8192-soft-byte frames, phase fix, derandomiser ("derandomize"), CCSDS C2 (8176, 7154) LDPC decoder, 1024-byte CADUs.
       "constellation": B200_BPSK / QPSK / OQPSK. Built: ldpc_rate 7. Device memory: about 7 bytes per max_soft byte (FIFO, fp32
       correlator scores, their syncword indices, decoder input, CADUs), so max_soft = 2^30 (the limit) takes about 7 GiB.            */
    int ldpc_rate;            /* 7 = "7/8" (C2). 1, 2, 4 = "1/2", "2/3", "4/5" (AR4JA): rejected                                         */
    int ldpc_block_size;      /* "ldpc_block_size" of the AR4JA codes (not built)                                                         */
    int ldpc_iterations;      /* "ldpc_iterations"                                                                                        */
    int ldpc2;                /* "ldpc2" (the labrador decoder): rejected                                                                 */
    int internal_stream;      /* "internal_stream": the 7136 info bits of every codeword go through BPSK_CCSDS_Deframer(internal_cadu_size,
                                 internal_asm) and its frames are the output (cadu_bytes = internal_cadu_size / 8; no RS)               */
    int internal_cadu_size;   /* "internal_cadu_size" bits, a multiple of 8 (frame padding is rejected); asm_sync carries "internal_asm"  */
    /* kind B200_FEC_TURBO = ccsds_turbo_decoder (module_ccsds_turbo_decoder.cpp:17-135): correlator on the rate's ASM (64, 96, 128 or 192
       bits) over frames of codeword + ASM soft bytes, derandomiser, CCSDS turbo decoder (log-MAP BCJR in double, deepspace-turbo), CRC-16;
       the frames whose CRC passes are written as 1A CF FC 1D + turbo_base bytes. All three fields are required. Device memory: about
       2.7 MB per frame of a decoding batch (at most 1024 frames) at turbo_base 1115, plus about 7 bytes per max_soft byte.              */
    int turbo_rate;           /* "turbo_rate": 2, 3, 4, 6 = "1/2", "1/3", "1/4", "1/6"                                                     */
    int turbo_base;           /* "turbo_base": 223, 446, 892 or 1115 (information bytes per frame)                                          */
    int turbo_iters;          /* "turbo_iters" >= 1 (the reference dereferences NULL with 0)                                               */
    /* kind B200_FEC_METOP_DUMP = metop_dump_decoder (no parameters): Correlator32 on the QPSK ASM 0x1ACFFC1D (8 syncwords: 4 phases x IQ
       swap, hard bits) over 8192-soft-byte frames, phase fix, hard decisions, inversion, derandomiser, RS(255,223) I=4 dual basis; every
       frame is written as 1A CF FC 1D + 1020 bytes, whatever RS returned. Only device and max_soft are read. Device memory: about 3 bytes
       per max_soft byte (FIFO, hard bits, correlator scores) plus 2 KiB of CADUs per 8192 soft bytes.                                 */
    /* kind B200_FEC_METEOR_LRPT = meteor_lrpt_decoder (module_meteor_lrpt_decoder.cpp:22-49), two modes:
       m2x_mode 0: Correlator on the 64-bit QPSK ASM (0xfca2b63db00d9794, or 0xfc4ef4fd0cc2df89 with diff_decode; 8 syncwords: 4 phases x
         IQ swap, hard bits) over 16384-soft-byte frames, phase fix, Viterbi27 (one r=1/2 k=7 CCDecoder of 8192 bits per frame, chained
         across frames), NRZ-M on the bytes when diff_decode, derandomiser, inversion when byte 9 is 0xFF, RS(255,223) I=4 in the
         conventional basis; the frames whose four codewords decode are written as 1D CF FC 1D + 1020 bytes. Only diff_decode, device
         and max_soft are read. Device memory: about 9 bytes per max_soft byte (FIFO, hard bits, correlator scores, the rotated frames,
         the Viterbi decisions), so max_soft = 2^28 (the limit) takes about 2.3 GiB.
       m2x_mode 1: the module's Viterbi1_2 (phases 0 and 90 degrees, IQ-swap check) -> NRZ-M bits when diff_decode -> BPSK_CCSDS_Deframer
         (8192) -> derandomiser -> RS(255,223) I=4 in the conventional basis, writing the frames whose four codewords decode: exactly
         ccsds_conv_concat_decoder with constellation "oqpsk", cadu_size 8192, nrzm = diff_decode, rs_i 4, rs_dualbasis false and
         rs_usecheck, and run by that decoder. outsync_after and ber_thresold are required ("viterbi_outsync_after",
         "viterbi_ber_thresold"). interleaved is refused (B200_EUNSUPPORTED): the reference's reader of that mode never delivers a
         sample, so there is no behaviour to reproduce. */
    int diff_decode;          /* "diff_decode" (required by the module)                                                                    */
    int m2x_mode;             /* "m2x_mode", default false                                                                                 */
    int interleaved;          /* "interleaved" (m2x_mode only), default false: refused                                                     */
    /* kind B200_FEC_NOAA_HRPT = noaa_hrpt_decoder (module_noaa_hrpt_decoder.cpp, noaa_deframer.cpp): hard bits soft > 0; the 60-bit
       minor-frame sync 0x0A116FD719D83C95 (or its complement: inverted) within deframer_thresold bits starts a frame, written as the
       six sync words 0x284 0x16F 0x35C 0x19D 0x20F 0x095 and 11084 10-bit words (MSB first, XOR the inversion). The output unit is ONE
       word: cadu_bytes = 2 (little-endian uint16, the .raw16 file), frames_out counts words (the module's frame_count = words / 11090),
       and a push writes every word whose 10th bit it brought. Only deframer_thresold, device and max_soft are read.
       kind B200_FEC_METEOR_HRPT = meteor_hrpt_decoder (module_meteor_hrpt_decoder.cpp, meteor/deframer.cpp): hard bits soft > 0 XOR the
       inversion; the ASM 0x1ACFFC1D machine with states 0 / 2 / 6 / 12 (each its own error threshold); every accepted ASM is followed by
       a frame written as 1A CF FC 1D + the next 8160 bits, returned when complete (cadu_bytes = 1024). Only device and max_soft are read.
       Both: device memory about 1.3 bytes per max_soft byte (FIFO, hard bits, sync bitmap) plus the output; max_soft <= 2^30. */
    /* kind B200_FEC_AQUA_DB = aqua_db_decoder (module_aqua_db_decoder.cpp:27-83, no parameters): per soft pair (I, Q) the QPSK hard symbol
       2*(Q>0) + (I>0); rail A = Q > 0, rail B = I > 0, each through its own NRZMDiff::decode_bits carried across pushes, interleaved A B A B
       -> BPSK_CCSDS_Deframer(8192, 0x1ACFFC1D) with its SYNCED state (and SYNCED error threshold) 10 instead of 12 -> derandomiser from
       byte 4 -> RS(255,223) I=4 dual basis; every frame is written as 1A CF FC 1D + 1020 bytes, whatever RS returned (cadu_bytes 1024).
       deframer_state reports 2 / 6 / 10. A push that ends inside a symbol keeps its odd byte for the next push. Only device and max_soft
       are read; max_soft <= 2^30. Device memory: about 1.4 bytes per max_soft byte (soft FIFO, bit FIFO, room for two pushes of CADUs). */
    int deframer_thresold;    /* "deframer_thresold" of noaa_hrpt_decoder (required by the module): 0 .. 60                              */
    /* kind B200_FEC_NOAA_GAC = noaa_gac_decoder (module_noaa_gac_decoder.cpp): hard bits soft > 0 -> BPSK_CCSDS_Deframer(33270, 0xA116FD71,
       backward: 0x33C3E4A6) with states 2 / 6 / 12 and 6 bits of padding: a frame is 4159 bytes, the clean sync word, the payload XOR the
       inversion, its last byte holding 6 bits right-aligned. backward reverses each frame's 33270 bits from that byte image, as the
       module does (the last two data bits are lost, two zero bits enter). Then every frame is XORed byte by byte with the GAC PN sequence
       (60 zero bits, then the 1023-bit sequence repeated). cadu_bytes 4159; backward playback's reversal of the frame ORDER is the file
       writer's (the host layer). Only backward, device and max_soft are read.
       kind B200_FEC_DMSP_RTD = dmsp_rtd_decoder (module_dmsp_rtd_decoder.cpp, dmsp_deframer.cpp): hard bits soft > 0 -> DMSP_Deframer(150, 2):
       the 13-bit sync 0b1010110011111 (or its complement: inverted), states 0 / 2 / 6, each its own error threshold; a frame is 19 bytes,
       the clean sync and 137 bits XOR the inversion, its last byte holding 6 bits right-aligned. Only device and max_soft are read.
       Both: max_soft <= 2^30; b200_fec_frame_bits returns the stream bit at which each pulled frame completed. */
    int backward;             /* "backward" of noaa_gac_decoder (required by the module): backward tape playback                         */
    /* kind B200_FEC_METEOR_XBAND = meteor_xband_decoder (module_meteor_xband_decoder.cpp): hard bits soft > 0 -> NRZMDiff::decode_bits
       carried across pushes, then by instrument_type:
         0 "mtvza": MTVZA_ExtDeframer (3072-bit records, four patterns) -> eight 46-byte packets XOR 0xAA per record ->
           SimpleDeframer(0x38FB456A, 32, 3040): one output unit is one 380-byte frame (cadu_bytes 380).
         1 "kmss_bpsk": RepackBitsByte -> KMSS_BPSK_ExtDeframer (1536-byte records) -> eight 188-byte packets per record -> three
           SimpleDeframers (syncs 0xAF5FFF50AA5AA0, 0xAE5EEC61BB7982, 0xAB5BB394EED628, 481280-bit frames) -> kmssFrameProcessor: one
           output unit is the four 15040-byte lanes of one frame (cadu_bytes 60160).
       Inner frames cut by the next sync are filled with zeros, as SimpleDeframer does. The decoder works in the module's 8192-byte reads
       counted from the stream's start: a push decodes every read it completes and keeps the rest, and the frames come out in the module's
       order (by read, then deframer, then position). Only instrument_type, device and max_soft are read; another instrument_type is
       refused ("Invalid METEOR instrument type!") before the device is looked at. max_soft <= 2^30. */
    int instrument_type;      /* "instrument_type": 0 "mtvza", 1 "kmss_bpsk"                                                              */
    /* kind B200_FEC_FENGYUN_AHRPT = fengyun_ahrpt_decoder (FengYun-3 AHRPT / DPT, module_fengyun_ahrpt_decoder.cpp): per 16384-byte read
       counted from the stream's start, the I/Q pairs swapped, I and Q split with the read's `shift` (0 or 1 symbol; the bytes past the
       read's end are 0) and Q complemented (~) when invert_second_viterbi, two Viterbi3_4 decoders in FengYun mode (8192 soft bytes ->
       6144 bits each; outsync_after, ber_thresold), the FengYun 2-bit differential decoder joining the two branches (swapped when the
       search machine says so), then, on reads where both Viterbis decoded, BPSK_CCSDS_Deframer(8192) with SYNCING 8 and SYNCED 16,
       the derandomiser from byte 4 and RS(255,223) I=4 dual basis; every frame is written whatever RS returned (cadu_bytes 1024).
       A push decodes every read it completes and keeps the rest. viterbi_state / viterbi_ber are viterbi1's, viterbi2_state /
       viterbi2_ber viterbi2's, deframer_state 2 / 8 / 16, rs_avg the last frame's. b200_fec_debug_fengyun_reads gives one record per
       read. max_soft <= 2^30. Device memory: about 7 bytes per max_soft byte (FIFO, the two branch streams, two Viterbi decisions).
       kind B200_FEC_FENGYUN_MPT = fengyun_mpt_decoder (FengYun-3 A/B/C MPT, module_fengyun_mpt_decoder.cpp): the same loop with two
       Viterbi1_2 decoders (phases 0 / 90, no I/Q-swap search; 8192 soft bytes -> 4096 bits each) in place of Viterbi3_4. The split is
       AHRPT's with Q always complemented, then each branch goes through rotate_soft(PHASE_0, swap): -128 -> -127 and the two bytes of
       every branch pair exchanged. Only a read that leaves viterbi1 in NOSYNC counts towards the shift toggle (the module tests viterbi1
       twice). The deframer has the default thresholds, deframer_state 2 / 6 / 12. The module has no invert_second_viterbi: a nonzero
       value is refused before the device is looked at. Stats, records and max_soft as for AHRPT. */
    int invert_second_viterbi; /* "invert_second_viterbi" (fengyun_ahrpt_decoder only; 0 for fengyun_mpt_decoder)                          */
} b200_fec_cfg;

typedef struct b200_demod_stats
{
    long samples_in, symbols_out;
    float agc_gain, costas_phase, costas_freq, mm_mu, mm_omega;
    long costas_unconverged;  /* junctions still inconsistent after the repair rounds of the last push (expected 0) */
    long mm_unconverged;      /* same for the M&M loop                                            */
    int agc_clamped;          /* batches so far in which the AGC hit max_gain (silent input): handled by the clamp pass */
    int repairs;              /* segments re-run as exact sequential continuations (junction check failed) */
    long kernel_launches;     /* CUDA kernels launched by this object so far                     */
    long agc_exact_passes;    /* batches whose AGC seeds needed the scanned (exact) pass: weak signal */
    long last_front_samples;  /* samples that entered the AGC in the last push (= nsamples unless the front-end resampler runs) */
    float snr, peak_snr;      /* M2M4SNREstimator over the recovered symbols, dB (module stats keys "snr" / "peak_snr", module_psk_demod.cpp:190-194,242-243):
                                 evaluated at the end of every push; the peak is the maximum of those */
    float pll_freq;           /* pm_demod: carrier PLL frequency, rad/sample (PLLCarrierTrackingBlock::getFreq; module stats key "freq" =
                                 rad_to_hz(pll_freq, final_samplerate), module_pm_demod.cpp:138,186) */
    long pll_unconverged;     /* pm_demod: carrier PLL junctions still inconsistent after the repair rounds of the last push (expected 0) */
    int repair_merge_hist[8]; /* the repairs by where they ended: [0] ran the whole segment; [i] met the segment's stored run at its
                                 checkpoint j (512 samples apart), 2^(i-2) < j <= 2^(i-1), and stopped there; [7]: any later one */
    int last_range_tiles;     /* 2048-sample tiles per range of the AGC + RRC kernel in the last push (b200_demod_debug_shape) */
} b200_demod_stats;

typedef struct b200_fec_stats
{
    long soft_in, chunks, bits_out, frames_out;
    int viterbi_state;        /* 0 NOSYNC 1 SYNCED  (Viterbi3_4::getState)                       */
    float viterbi_ber;
    int deframer_state;       /* 2 NOSYNC / 6 SYNCING / 12|18 SYNCED (BPSK_CCSDS_Deframer; aqua_db_decoder: 10); meteor_hrpt_decoder: its own state
                                 numbers 0 (NOSYNC) / 2, 6 (SYNCING) / 12 (SYNCED, "deframer_lock"); noaa_hrpt_decoder: 0;
                                 noaa_gac_decoder: 2 / 6 / 12; dmsp_rtd_decoder: 0 (NOSYNC) / 2 (SYNCING) / 6 (SYNCED)                */
    long rs_corrected, rs_failed;
    long replays;             /* slow-path re-decodes (lock changes, start-state mis-speculation) */
    long kernel_launches;
    long start_redone;        /* chunks decoded again because their speculated Viterbi start state was wrong (part of replays) */
    long tb_serial;           /* chunks whose parallel chainback blocks disagreed and were chained back serially (part of replays) */
    int spec_steps;           /* current length of the start-state speculation window (adapts to the channel) */
    int tb_overlap;           /* current warm-up length of the parallel chainback blocks (adapts to the channel) */
    /* ccsds_ldpc_decoder (module stats keys, module_ccsds_ldpc_decoder.cpp:279-295), of the last frame decoded */
    int correlator_lock;      /* "correlator_lock": the ASM was found at the expected place (pos 0); "lock_state" SYNCED / NOSYNC.
                                 internal_stream: deframer_state above is "deframer_state" (deframer_lock = SYNCED)                   */
    float correlator_corr;    /* "correlator_corr": the correlator's best score                                                       */
    int ldpc_corr;            /* "ldpc_corr": info positions whose decoded bit differs from the sign of the input                     */
    long ldpc_resyncs;        /* frames so far whose ASM was not at the expected place (the frame walk shifted)                       */
    /* ccsds_turbo_decoder: correlator_lock / correlator_corr above are its "Corr" and lock state; ldpc_resyncs counts its shifted frames.
       metop_dump_decoder: correlator_lock is "lock_state" (SYNCED iff the last frame's pos was 0), correlator_corr its correlation (0..32),
       ldpc_resyncs the frames whose pos was not 0, rs_corrected / rs_failed above its RS results */
    long crc_ok, crc_fail;    /* frames so far whose CRC-16 passed (written) / failed ("CRC Check" PASS / FAIL)                        */
    long turbo_near_ties;     /* decisions so far whose margin |one - zero| was below 1e-9 (where libm rounding could tip a bit)       */
    /* meteor_lrpt_decoder: "rs_avg" = (errors[0] + errors[1] + errors[2] + errors[3]) / 4 of the last frame decoded (0 before the first).
       m2x_mode 0: correlator_lock ("correlator_lock", "lock_state"), correlator_corr (0..64), ldpc_resyncs (frames whose pos was not 0),
       viterbi_ber (Viterbi27's BER of the last frame) and rs_corrected / rs_failed above; m2x_mode 1: the keys of
       ccsds_conv_concat_decoder above */
    int rs_avg;
    int viterbi2_state;       /* fengyun_ahrpt / _mpt_decoder: "viterbi2_lock" (viterbi_state above is "viterbi1_lock")                */
    float viterbi2_ber;       /* fengyun_ahrpt / _mpt_decoder: "viterbi2_ber" (viterbi_ber above is "viterbi1_ber")                   */
} b200_fec_stats;

typedef struct b200_demod b200_demod;

/* BaseDemodModule::initb's choice of the working sample rate (module_demod_base.cpp:59-87): returns samplerate when
 * samplerate/symbolrate lies inside [min_sps, max_sps] (psk_demod: 1.1..4.0, OQPSK 1.6..2.4; pass 0 for those defaults), else the
 * rate the reference's front-end resampler converts to. custom_samplerate > 0 overrides ("custom_samplerate"). */
double b200_demod_final_samplerate(double samplerate, double symbolrate, int constellation, float min_sps, float max_sps, double custom_samplerate);
/* BaseDemodModule::initb's `resample` (module_demod_base.cpp:66): 1 when samplerate / symbolrate lies outside [min_sps, max_sps] */
int b200_demod_resample_decision(double samplerate, double symbolrate, int constellation, float min_sps, float max_sps);
/* The polyphase bank the front-end resampler uses for (samplerate -> final_samplerate): RationalResamplerBlock::set_ratio
 * (resamp/rational_resampler.cpp:27-41) = firdes::design_resampler_filter_float + PolyphaseBank::init. Host-only (no device):
 * out[arm * *ntaps + k], *interp arms, reduced ratio *interp / *decim. */
int b200_demod_resampler_bank(double samplerate, double final_samplerate, float *out, long cap, int *ntaps, int *interp, int *decim);
typedef struct b200_fec b200_fec;
typedef struct b200_chain b200_chain;

const char *b200_last_error(void);
int b200_device_count(void);

/* ---- demodulator: raw IQ -> soft symbols ---------------------------------------------------------- */
b200_demod *b200_demod_create(const b200_demod_cfg *cfg);
void b200_demod_destroy(b200_demod *d);
/* One batch of the stream from HOST memory (copied to the device inside the call). Loop state carries over. */
int b200_demod_push_iq(b200_demod *d, const void *host_iq, long nsamples);
/* Same, samples already in device memory of cfg.device (no copy). */
int b200_demod_push_iq_device(b200_demod *d, const void *dev_iq, long nsamples);
/* int8 soft symbols of the LAST push (I,Q interleaved; BPSK: I only) — the bytes PSKDemodModule writes to .soft / the FIFO */
int b200_demod_pull_soft(b200_demod *d, int8_t *host_out, long cap, long *n_out);
/* float symbols of the LAST push (M&M output, interleaved re,im; fsk_demod: one float per symbol) */
int b200_demod_pull_symbols(b200_demod *d, float *host_out, long cap_symbols, long *n_out);
/* stage outputs of the LAST push (needs keep_stages): nsamples complex values, interleaved re,im */
int b200_demod_debug_stage(b200_demod *d, int stage, float *host_out, long cap_samples);
/* Stage-isolated parity hook (SURVEY.md 8c): runs ONE stage of a freshly reset demodulator on a caller-supplied stage input
 * (nsamples complex values, interleaved re,im: normally the ORACLE's output of the stage before) and returns the stage output.
 *   B200_STAGE_FIR     in = AGC output.  mode STRICT: fir.cpp:74-83 in the generic VOLK order -> bitwise the oracle's FIR output;
 *                      mode 0: the production kernel (k_agc_fir_w with the AGC switched off), one fma per tap
 *   B200_STAGE_COSTAS  in = FIR output; out = what the clock recovery reads (rotation fix-up, OQPSK delay, post_costas_dc applied)
 *   B200_STAGE_MM      in = the clock recovery's input; out = symbols (*n_out of them). STRICT | SEQUENTIAL -> bitwise the oracle's
 * fsk_demod: B200_STAGE_QUAD (in = complex AGC output), DC2, AGC2, FIR and MM (in = the previous stage's output): one float per sample
 *   in and out (QUAD: complex in). QUAD and FIR are always the reference's arithmetic; DC2 and AGC2 with SEQUENTIAL run the recurrence as
 *   one float thread, MM as above.
 * SEQUENTIAL runs the loop as one segment (no warm-up, no stitching). The demodulator is reset before and after. */
int b200_demod_debug_run_stage(b200_demod *d, int stage, const float *host_in, long nsamples, int mode, float *host_out, long cap_complex, long *n_out);
/* Junction residuals of the LAST push / debug run: per segment s > 0 the Costas phase (mod 2pi/order) and frequency difference
 * between segment s's warmed-up state at its first owned sample and segment s-1's end state (costas_out[2s], [2s+1]), and the M&M
 * sampling-instant difference (mm_out[s], samples). Either pointer may be NULL. */
int b200_demod_debug_junctions(b200_demod *d, double *costas_out, double *mm_out, long cap_segments, long *nseg_out, long *seg_len);
/* test hook: only the sample conversion (BasebandReader::read_samples, baseband_interface.h:170-190) of `nsamples` host samples */
int b200_demod_debug_convert(b200_demod *d, const void *host_iq, long nsamples, float *host_out);
/* test hook: enable = 0 gives the repairs a tolerance of 0 for meeting the stored run, so every repair runs its whole segment */
int b200_demod_debug_repair_merge(b200_demod *d, int enable);
/* test hook: the shape of this handle's pushes, so that tests reach the geometries of large pushes with small ones.
 *   range_tiles > 0: the AGC + RRC kernel runs ranges of that many 2048-sample tiles (0: the production rule, at least 4 tiles; the
 *                    floor only amortises the walk back that proves each range's start gain, any length >= 1 computes the same stream)
 *   seg_len > 0:     the loop kernels' segment length, a multiple of 16 in [4096, 16384] (0: the production rule); else B200_EINVAL
 *   keep_front != 0: each push copies the production front kernel's RRC output, so that b200_demod_debug_stage(B200_STAGE_FIR)
 *                    returns it. A keep_stages handle runs the dumping variant of that kernel instead and refuses this.
 * The range length of the last push is b200_demod_stats.last_range_tiles, its segment length b200_demod_debug_junctions' seg_len. */
int b200_demod_debug_shape(b200_demod *d, int range_tiles, int seg_len, int keep_front);
/* Cycle counters of the loop kernels' main passes, only in a library built with -DB200_LOOP_CYCLES (tools/profile_loops.py --cycles):
 * out[0..3] = clock64() cycles summed over the warps of k_costas (or k_pll) in its phases row wait, loop, copy-out, tail, out[4] = those
 * warps; out[5..9] the same for k_mm (row wait, input fix-up, symbol loop, symbol copy-out; warps), all since the previous call, which
 * they clear. cap >= 10. A production library returns B200_EUNSUPPORTED. */
int b200_demod_debug_loop_cycles(unsigned long long *out, int cap);
int b200_demod_get_stats(b200_demod *d, b200_demod_stats *out);
/* forget the stream (loop state, resampler counters) but keep every allocation: the next push starts a new stream */
int b200_demod_reset(b200_demod *d);
/* double buffering for host streams, as b200_chain_prefetch_iq: start the H2D copy of a FUTURE batch (pinned memory); the later
 * b200_demod_push_iq() with the same (pointer, nsamples) only waits for it */
int b200_demod_prefetch_iq(b200_demod *d, const void *host_iq, long nsamples);
/* elapsed device milliseconds of the last push (CUDA events on the demodulator's stream): [0] = sum, [1] = (front end +) AGC + FIR,
 * [2] = Costas + rotation (+ OQPSK delay), [3] = M&M + compaction / quantiser */
int b200_demod_last_timing(b200_demod *d, float *ms_out, int n);
/* RRC taps / M&M polyphase bank as designed on the host (for parity tests against firdes / PolyphaseBank) */
int b200_demod_get_taps(b200_demod *d, float *rrc_out, int rrc_cap, float *bank_out /* 128*8 or NULL */);

/* ---- decoder: soft symbols -> CADUs --------------------------------------------------------------- */
b200_fec *b200_fec_create(const b200_fec_cfg *cfg);
void b200_fec_destroy(b200_fec *f);
int b200_fec_push_soft(b200_fec *f, const int8_t *host_soft, long n);
int b200_fec_push_soft_device(b200_fec *f, const int8_t *dev_soft, long n);
/* frames completed by the pushes since the last pull, cadu_bytes each, in stream order */
int b200_fec_pull_frames(b200_fec *f, uint8_t *host_out, long cap, long *nbytes_out);
/* Viterbi output bits (1 bit per byte, after NRZ-M when enabled) of the LAST push, for stage tests */
int b200_fec_debug_bits(b200_fec *f, uint8_t *host_out, long cap, long *n_out);
int b200_fec_get_stats(b200_fec *f, b200_fec_stats *out);
int b200_fec_cadu_bytes(b200_fec *f);
int b200_fec_chunk_size(b200_fec *f);
/* ccsds_ldpc_decoder: one record per frame of the LAST push, in stream order */
typedef struct b200_ldpc_frame
{
    long offset;              /* stream offset (soft bytes since create / reset) of the frame's first byte                           */
    int pos;                  /* the correlator's position in the window read before it (0 = locked)                                */
    float cor;                /* correlator_corr                                                                                    */
    int phase, swap;          /* the phase ambiguity fixed (0..3 = 0, 90, 180, 270 degrees) and the OQPSK re-delay / IQ swap         */
    int ldpc_corr;
} b200_ldpc_frame;
int b200_fec_debug_ldpc_frames(b200_fec *f, b200_ldpc_frame *out, long cap, long *n_out);
/* ccsds_ldpc_decoder only (B200_EINVAL for the other kinds): elapsed device milliseconds of the last push (CUDA events on the decoder's
   stream): [0] correlation, [1] frame walk, [2] gather, [3] decode + CADU repack (+ internal_stream: bit append, deframer, frames),
   [4] the whole push */
int b200_fec_ldpc_timing(b200_fec *f, float *ms_out, int n);
/* ccsds_turbo_decoder: one record per frame of the LAST push, in stream order (frames whose CRC fails included) */
typedef struct b200_turbo_frame
{
    long offset;              /* stream offset (soft bytes since create / reset) of the frame's first byte                           */
    int pos;                  /* the correlator's position in the window read before it (0 = locked)                                */
    float cor;                /* the correlator's best score ("Corr")                                                               */
    int swapped;              /* the ASM correlated negatively: the soft bits were negated                                          */
    int crc_ok;               /* the CRC-16 passed and the frame was written                                                        */
} b200_turbo_frame;
int b200_fec_debug_turbo_frames(b200_fec *f, b200_turbo_frame *out, long cap, long *n_out);
/* ccsds_turbo_decoder: the a-priori arrays (log-domain, input 0 and input 1, in information-bit order) that frame `frame` of the LAST push
   held after its last iteration, 8 turbo_base values each: turbo_decode's `messages` after the final message_deinterleave. Frames of the
   push's last decoding batch only (the last 1024 frames). */
int b200_fec_debug_turbo_llr(b200_fec *f, long frame, double *app0, double *app1, long cap, long *n_out);
/* ccsds_turbo_decoder only (B200_EINVAL for the other kinds): elapsed device milliseconds of the last push: [0] correlation, [1] frame
   walk, [2] gather, [3] BCJR iterations, [4] packing, CRC and compaction, [5] the whole push */
int b200_fec_turbo_timing(b200_fec *f, float *ms_out, int n);
/* metop_dump_decoder: one record per frame of the LAST push, in stream order */
typedef struct b200_dump_frame
{
    long offset;              /* stream offset (soft bytes since create / reset) of the frame's first byte (after the shift)          */
    int pos;                  /* the correlator's position in the window read before it (0 = locked; >= 8192: a window-tail winner,
                                 which the module does not shift)                                                                   */
    int corr;                 /* the correlator's value (0..32)                                                                    */
    int phase, swap;          /* the phase ambiguity fixed (0..3 = 0, 90, 180, 270 degrees) and the IQ swap                        */
    int rs[4];                /* decode_interlaved's errors[] of the four codewords: -1 = not decodable, else bytes corrected       */
} b200_dump_frame;
int b200_fec_debug_dump_frames(b200_fec *f, b200_dump_frame *out, long cap, long *n_out);
/* meteor_lrpt_decoder with m2x_mode 0: one record per frame of the LAST push, in stream order (frames dropped by RS included) */
typedef struct b200_meteor_frame
{
    long offset;              /* stream offset (soft bytes since create / reset) of the frame's first byte (after the shift)          */
    int pos;                  /* the correlator's position in the window read before it (0 = locked)                                */
    int corr;                 /* the correlator's value (0..64)                                                                    */
    int phase, swap;          /* the phase ambiguity fixed (0..3 = 0, 90, 180, 270 degrees) and the IQ swap                        */
    int rs[4];                /* decode_interlaved's errors[] of the four codewords: -1 = not decodable, else bytes corrected       */
    float ber;                /* Viterbi27's BER of the frame                                                                      */
} b200_meteor_frame;
int b200_fec_debug_meteor_frames(b200_fec *f, b200_meteor_frame *out, long cap, long *n_out);
/* noaa_hrpt_decoder / meteor_hrpt_decoder: one record per sync accepted in the LAST push, in stream order (frames still open included) */
typedef struct b200_hrpt_frame
{
    long bit;                 /* stream bit index (soft bytes since create / reset) of the sync's last bit                            */
    int inverted;             /* the frame is written inverted (the sync's complement matched)                                       */
    int state;                /* the state that accepted it: METEOR 0 / 2 / 6 / 12; NOAA 0                                            */
} b200_hrpt_frame;
int b200_fec_debug_hrpt_frames(b200_fec *f, b200_hrpt_frame *out, long cap, long *n_out);
/* noaa_gac_decoder / dmsp_rtd_decoder: for each frame the last b200_fec_pull_frames returned, in order, the stream bit index (soft bytes
   since create / reset) of the bit that completed it. dmsp_rtd_decoder's "_timestamps.txt" needs it: the module stamps a frame with the
   number of 8192-byte reads that produced frames, up to the one holding that bit. Other kinds: B200_EINVAL. */
int b200_fec_frame_bits(b200_fec *f, long *out, long cap, long *n_out);
/* fengyun_ahrpt_decoder / fengyun_mpt_decoder: one record per 16384-byte read the LAST push completed, the module's variables at the end
   of that read */
typedef struct b200_fengyun_read
{
    long read;                /* read index since create / reset                                                                      */
    int shift, invert_branches; /* the search machines after the read (shift toggles after 10 reads with a Viterbi in NOSYNC; the
                                 branches swap after 10 deframer NOSYNC reads)                                                        */
    int v1, v2;               /* bits each Viterbi returned: 0 or 6144 (AHRPT) / 4096 (MPT)                                           */
    int state1, state2;       /* Viterbi3_4 / Viterbi1_2::getState() after the read: 0 NOSYNC, 1 SYNCED                                */
    float ber1, ber2;         /* Viterbi3_4 / Viterbi1_2::ber() after the read                                                        */
    int deframer_state;       /* 2 / 8 / 16 (AHRPT) or 2 / 6 / 12 (MPT) after the read                                                */
    int pad;
} b200_fengyun_read;
int b200_fec_debug_fengyun_reads(b200_fec *f, b200_fengyun_read *out, long cap, long *n_out);

/* ---- fused chain: raw IQ -> CADUs, soft stream stays in HBM ---------------------------------------- */
b200_chain *b200_chain_create(const b200_demod_cfg *dcfg, const b200_fec_cfg *fcfg);
void b200_chain_destroy(b200_chain *c);
int b200_chain_push_iq(b200_chain *c, const void *host_iq, long nsamples);
int b200_chain_push_iq_device(b200_chain *c, const void *dev_iq, long nsamples);
/* Double buffering for host streams: start the H2D copy of a FUTURE batch (pinned memory) on a copy stream; the later
 * b200_chain_push_iq() with the same (pointer, nsamples) only waits for it. At most two batches may be pending. */
int b200_chain_prefetch_iq(b200_chain *c, const void *host_iq, long nsamples);
int b200_chain_pull_frames(b200_chain *c, uint8_t *host_out, long cap, long *nbytes_out);
/* device-resident result access (no D2H): pointer to the frames produced since the last pull/reset */
int b200_chain_frames_device(b200_chain *c, const uint8_t **dev_ptr, long *nbytes);
int b200_chain_get_stats(b200_chain *c, b200_demod_stats *ds, b200_fec_stats *fs);
/* timing taps used by bench.py: elapsed device milliseconds of the last push per stage (CUDA events on the chain's stream) */
int b200_chain_last_timing(b200_chain *c, float *ms_out, int n); /* n >= 9: [0]=sum of stages [1]=agc+fir [2]=costas(+rotate) [3]=m&m [4]=viterbi stage [5]=deframe+rs [6]=k_vit_main alone [7]=chunks it decoded [8]=whole push, event timed */
/* forget the stream (loop state, lock, FIFOs) but keep every allocation: the next push starts a new stream */
int b200_chain_reset(b200_chain *c);
/* Pipelined mode: the decoder runs on a worker thread and its own CUDA stream one batch behind the demodulator, like the
 * reference's one-thread-per-module pipeline (src-core/pipeline/pipeline_run.cpp:44-117) with a whole batch of soft symbols in HBM
 * as the FIFO element. push(i) returns when batch i is demodulated and batch i-1 decoded; b200_chain_pull_frames() then returns
 * the frames of the batches decoded so far without waiting for the one in flight; b200_chain_sync() waits for the decoder
 * (after it, pull returns everything). Decoder errors surface at the next push / sync. Output is identical to the synchronous mode. */
int b200_chain_set_pipelined(b200_chain *c, int on);
int b200_chain_sync(b200_chain *c);
/* CUDA-event stopwatch over several pushes (both streams): begin syncs the chain and stamps the demodulator's stream, end syncs
 * and stamps the decoder's stream; *ms = elapsed device time */
int b200_chain_span_begin(b200_chain *c);
int b200_chain_span_end(b200_chain *c, float *ms);

/* ---- CADU -> CCSDS space packets (the step behind the decoder; SURVEY 8f row 3) --------------------------------------------
 * Replaces, for all selected virtual channels at once, what the instrument modules do per CADU on the host
 * (plugins/noaa_metop_support/metop/module_metop_instruments.cpp:66-140): ccsds::ccsds_aos::parseVCDU(cadu).vcid
 * (src-core/common/ccsds/ccsds_aos/vcdu.cpp:10-17) selects one ccsds::ccsds_aos::Demuxer per channel, whose work(cadu)
 * (ccsds_aos/demuxer.cpp:64-199; M-PDU header mpdu.cpp:9-13) returns the space packets completed by that frame. The packets come
 * back in exactly that order - frame by frame, inside a frame in the order work() returns them - with exactly the reference's bytes,
 * including its behaviour on inconsistent frames. */
typedef struct b200_demux_cfg
{
    int cadu_size;                /* bytes per CADU as the decoder writes them (1024 for RS interleaving 4)                          */
    int mpdu_data_size;           /* Demuxer(mpdu_data_size, ...), demuxer.h:33 (default 884; MetOp: 882 with a 2-byte insert zone)  */
    int has_insert_zone;          /* Demuxer(.., hasInsertZone, insertZoneSize, ..)                                                  */
    int insert_zone_size;
    int secondary_header_extends; /* Demuxer(.., secondaryHeaderExtendsPkt): + 8 payload bytes when the secondary header flag is set */
    unsigned long long vcid_mask; /* bit v set = virtual channel v is demultiplexed (the modules' `if (vcdu.vcid == N)` chains)      */
    int device;
    long max_frames;              /* largest number of CADUs of one push                                                             */
    long max_packets;             /* room of the packet table of one push; 0 = 8 * max_frames + 1024                                 */
} b200_demux_cfg;
typedef struct b200_packet
{
    long offset;      /* of the packet's 6 header bytes (CCSDSHeader::raw) in the byte stream of the pull; payload behind them      */
    int payload_len;  /* CCSDSPacket::payload.size()                                                                                */
    int frame;        /* stream index (since create / reset) of the CADU whose work() call returned the packet                      */
    short vcid, apid; /* parseVCDU(cadu).vcid; CCSDSHeader::apid                                                                    */
} b200_packet;
typedef struct b200_demux_stats
{
    long frames_in, packets_out, kernel_launches;
    long redone_channels; /* virtual channels walked a second time, serially, because leftover bytes of an unfinished packet crossed a window
                             boundary of the parallel walk (inconsistent frames only; expected 0) */
} b200_demux_stats;
typedef struct b200_demuxer b200_demuxer;
b200_demuxer *b200_demux_create(const b200_demux_cfg *cfg);
void b200_demux_destroy(b200_demuxer *d);
/* nframes CADUs of cadu_size bytes from host memory / already on the device (e.g. b200_chain_frames_device) */
int b200_demux_push_frames(b200_demuxer *d, const uint8_t *host_cadus, long nframes);
int b200_demux_push_frames_device(b200_demuxer *d, const uint8_t *dev_cadus, long nframes);
/* packets of the LAST push: `bytes` = [6 header bytes][payload] back to back, `packets` = one record each */
int b200_demux_pull(b200_demuxer *d, uint8_t *bytes, long cap_bytes, long *nbytes, b200_packet *packets, long cap_packets, long *npackets);
int b200_demux_reset(b200_demuxer *d);
int b200_demux_get_stats(b200_demuxer *d, b200_demux_stats *out);

#ifdef __cplusplus
}
#endif
#endif
