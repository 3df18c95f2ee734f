// Host side of the demodulator: owns the device buffers / carried loop state of ONE baseband stream and launches
// the kernels of demod.cuh for each pushed batch. Mirrors what PSKDemodModule::init() builds
// (src-core/pipeline/modules/demod/module_psk_demod.cpp:86-136, module_demod_base.cpp:59-208).
#pragma once
#include "demod.cuh"
#include "host_common.h"
#include <vector>

namespace b200
{

// carried loop state, double buffered by batch parity (kernels read [cur], write [cur^1])
struct DemodDevState
{
    float gain[2];
    float costas[2][2]; // phase, freq
    MMState mm[2];
    float2 agc_tail[2][32];
    float2 rs_tail[2][RS_MAX_TAPS]; // resampler history (ntaps-1 converted input samples)
    float2 dc_acc[2];               // DC blocker accumulator (correct_iq.h: acc)
    float2 dc_acc2[2];              // accumulator of the post-Costas DC blocker
    float2 pdc_hist[2][MM_HIST];    // its last outputs: the clock recovery's history across batches
    float2 mm_hist[2][MM_HIST];
    int flags;          // bit0 AGC clamp, bit1 M&M slot overflow
    int costas_unconv;  // junctions still unconverged after the repair rounds of the last batch
    int mm_unconv;
    int repairs;        // segments re-run as exact continuations so far (all batches)
    int merge_hist[MERGE_BUCKETS]; // ... by the checkpoint at which the re-run met the stored run and stopped (count_repair)
    int agc_exact;      // batches that needed the exact AGC pass so far
    float snr_y[2][2];  // M2M4 SNR estimator: running averages of |s|^2, |s|^4 (snr_estimator.h:26)
    // pm_demod (module_pm_demod.cpp:61-88)
    float pll[2][2];           // carrier PLL phase, frequency (pll_carrier_tracking.h: d_phase, d_freq)
    float gain2[2];            // the AGC in front of the RRC: AGCBlock(0.001, 1, 1, 1000) with resample_after_pll, else the identity (rate 0, gain 1)
    float2 agc2_tail[2][32];   // ... and its FIR history
    float2 agc1_tail[2][32];   // (the first AGC's kernel also keeps a FIR history; unused in pm mode)
    int pll_unconv;            // carrier PLL junctions still unconverged after the repair rounds of the last batch
    float2 dc_acc3[2];         // psk_demod carrier mode: accumulator of the DC blocker behind the carrier PLL (module_psk_demod.cpp:112)
    // fsk_demod (module_fsk_demod.cpp:59-84)
    float qphase[2];           // QuadratureDemodBlock::phase: p of the last sample
    float fdc_acc[2];          // CorrectIQBlock<float>::acc
    float fgain[2];            // AGCBlock<float>::gain
    float fir_tail[2][32];     // the FIRBlock<float> history: the AGC's last 32 outputs
};

// one AGC (+ RRC) pass of k_agc_fir_w: which carried gain / FIR history it uses and where its outputs go
struct AgcUnit
{
    float rate, max_gain;
    float *gain_in, *gain_out;
    const float2 *tail_in;
    float2 *tail_out, *fir_out, *dump; // dump != nullptr: also write the AGC output there
};

class Demod
{
  public:
    explicit Demod(const b200_demod_cfg &cfg);
    ~Demod();
    // Processes one batch already resident on the device. If soft_dst != nullptr the int8 soft symbols are appended
    // there (device pointer), otherwise into the object's own soft buffer. Returns the number of symbols produced.
    long process(const void *d_raw, long nsamples, int8_t *soft_dst);
    long push_host(const void *h_raw, long nsamples, int8_t *soft_dst);
    // Starts the host->device copy of a FUTURE batch on a dedicated copy stream (double buffered); the matching push_host()
    // then only waits for that copy. Lets the H2D of batch i+1 overlap the kernels of batch i. Pinned host memory required.
    void prefetch_host(const void *h_raw, long nsamples);
    void stats(b200_demod_stats *out);
    void reset(); // back to the state of a freshly created demodulator (new stream)
    void init_state(); // the initial DemodDevState, into h_state and (on the stream) st
    // stages of process(), also run alone by the stage-isolated parity hook
    float2 *stage_costas(long n, int L, int nseg, int cur, int nxt, bool materialise);
    // front-end resampler (power-of-two decimator stages + rational resampler) over n samples at d_raw: updates them to its output
    void front_resample(const void *&d_raw, long &n, int &front_fmt, int &rs_swap, long n_in, int cur, int nxt);
    // pm_demod: carrier PLL over n AGC'd samples (pm_agc -> pm_pll), then PMToBPSK (-> pm_out)
    void stage_pll(long n, int cur, int nxt);
    // PLLCarrierTrackingBlock (segmented, junction check + repair rounds) over n samples: in -> out
    void run_pll(const float2 *in, float2 *out, long n, float bw, float max_offset, int cur, int nxt);
    void run_rotator(const void *src, int fmt, long n, int iq_swap, int imag_only, unsigned long long dturn, unsigned long long pos, float2 *dst);
    // CorrectIQBlock over n samples: src -> dst, carried accumulator acc_in -> acc_out
    void run_dc(const void *src, int fmt, int iq_swap, long n, const float2 *acc_in, float2 *acc_out, float2 *dst);
    const uint8_t *mm_quad = nullptr; // set by stage_costas when the clock recovery applies the rotation (/ OQPSK delay) itself
    int mm_rot = 0, mm_oqpsk = 0;
    void stage_mm(float2 *mmin, long n, int L, int nseg, int cur, int nxt, int8_t *sdst, bool strict, bool all_symbols);
    long debug_run_stage(int stage, const float *h_in, long n, int mode, float *h_out, long cap);
    long debug_run_stage_fsk(int stage, const float *h_in, long n, int mode, float *h_out, long cap);
    int last_L = 0, last_nseg = 0;          // segmentation of the last batch (b200_demod_debug_junctions)
    int dbg_costas_unconv = 0, dbg_mm_unconv = 0, dbg_repairs = 0; // of the last debug_run_stage
    // junction tolerances: Costas phase (rad) / frequency (rad/sample) residual, M&M sampling instant (samples)
    float tol_cphase = 2e-3f, tol_cfreq = 1e-4f, tol_mm = 0.05f;
    float tol_momega = 0.f;    // M&M omega (samples per symbol): only a repair that joins the stored run checks it
    // A repair stops at a checkpoint where it agrees with the stored run within 1 / MERGE_TIGHTER of the junction tolerances: the end
    // record it keeps then differs from the exact continuation's by so little that no junction check of the successor comes out
    // differently (measured on the 6-samples-per-symbol pm_demod signal, where the M&M runs approach each other slowly: with the
    // junction tolerance itself 5 of 510 repairs of successors no longer happen, with 1/2 and 1/4 one, from 1/8 on none).
    static constexpr float MERGE_TIGHTER = 16.0f;
    bool repair_merge = true;  // test hook (b200_demod_debug_repair_merge): false = tolerance 0, every repair runs its whole segment
    // test hook (b200_demod_debug_shape): forced range length of k_agc_fir_w / segment length of the loop kernels (0: production
    // rules), and a copy of the production front kernel's RRC output into fir_dump
    int dbg_range_tiles = 0, dbg_seg_len = 0;
    bool keep_front = false;
    int last_R = 0; // range length of the last launch_front

    b200_demod_cfg cfg;
    cudaStream_t stream = nullptr;
    int bps;       // soft bytes per symbol (1 BPSK, else 2)
    int order;     // Costas order, 0 = none
    float sps;
    std::vector<float> rrc, bank;
    long last_n = 0, last_syms = 0;
    long total_in = 0, total_syms = 0, launches = 0;
    int parity = 0;
    float t_agcfir = 0, t_costas = 0, t_mm = 0; // ms of the last batch
    DevBuf<unsigned char> raw, raw2;
    cudaStream_t copy_stream = nullptr;
    struct Prefetch { const void *ptr = nullptr; long n = 0; int buf = 0; bool valid = false; cudaEvent_t done = nullptr; long seq = 0; } pf[2];
    long pf_seq = 0;
    DevBuf<float2> bufA, bufB, agc_dump, fir_dump, slots, sym_out;
    DevBuf<int8_t> soft;
    DevBuf<Affine3> tile_map3;     // clamp pass (silent input): per-tile maps with the max_gain clamp
    long agc_clamped_batches = 0;
    DevBuf<Affine> tile_map;       // exact AGC pass (weak signals): per-tile maps,
    DevBuf<double> seeds;          // gain before every tile
    DevBuf<int> agc_need;          // [2] raised by the fast pass when a range cannot prove its seed
    unsigned agc_epoch = 0;
    int fir_ctas = 0;              // resident k_agc_fir_w CTAs on the device
    int fir_warps = 0;             // ... and their warps: one range of tiles each (one wave)
    // front-end resampler (RationalResamplerBlock) / iq_swap pass
    bool resamp = false;
    int rs_I = 1, rs_D = 1, rs_nt = 1;
    long rs_inc = 0, rs_ctr = 0;   // carried counters (rational_resampler.h: inc, d_ctr)
    std::vector<float> rs_bank;
    DevBuf<float> d_rs_bank;
    DevBuf<float2> rs_out;
    // power-of-two decimator in front of the rational resampler (SmartResamplerBlock with samplerate / final_samplerate >= 2)
    struct DecimStage
    {
        int D = 1, nt = 0;
        long inc = 0;                  // carried decimation phase (decimating_fir.h: inc)
        std::vector<float> taps_rev;
        DevBuf<float> d_taps;
        DevBuf<float2> tail[2], out;   // last nt - 1 inputs by batch parity; stage output (cf32)
        DecimStage() = default;
        DecimStage(DecimStage &&o) noexcept : D(o.D), nt(o.nt), inc(o.inc), taps_rev(std::move(o.taps_rev)) {}
    };
    std::vector<DecimStage> decim;
    int decim_total = 1;
    long max_work = 0;             // largest sample count after the front end
    DevBuf<DcAff> dc_map;          // DC blocker: per-tile maps, per-tile accumulators, output (cf32)
    DevBuf<double2> dc_seeds;
    DevBuf<float2> dc_out;
    DevBuf<float2> pdc_out;        // post-Costas DC blocker output (16-sample front pad like bufA / bufB)
    long last_front = 0;           // samples that entered the AGC in the last batch
    long last_in = 0;              // samples pushed in the last batch
    int agc_warm_max = 24;
    DevBuf<LoopRec> crec;
    DevBuf<MMRec> mrec;
    DevBuf<LoopCkpt> cck; // repair checkpoints of the last phase-loop / clock-recovery stage: ckpt_per_seg(L) per segment
    DevBuf<MMCkpt> mck;
    DevBuf<uint8_t> quad;
    DevBuf<int> repair; // [0] count, [1..1024] junction list (shared by the Costas and M&M repair rounds)
    DevBuf<long> offs;
    DevBuf<float> d_bank;
    DevBuf<DemodDevState> st;
    PinnedBuf<long> h_total;
    PinnedBuf<DemodDevState> h_state; // snapshot for stats
    cudaEvent_t ev[4];
    int Wc, Wm, Gc = 0, Gm = 0, seg_cap_threads; // warm-up lengths, gear-shift parts of them
    // pm_demod / freq_shift
    bool pm = false, pm_after = false;   // PMDemodModule's chain; its resampler sits behind the PLL ("resample_after_pll")
    int Wp = 0;                          // carrier PLL warm-up
    float tol_pphase = 1e-5f, tol_pfreq = 2e-6f;
    unsigned long long pm_dturn = 0, fs_dturn = 0; // rotator steps of PMToBPSK / FreqShiftBlock: fraction of a turn per sample, 0.64 fixed point
    unsigned long long pm_pos = 0, fs_pos = 0;     // samples those rotators have seen so far
    DevBuf<float2> pm_agc, pm_pll, pm_out, fs_out; // (pm_agc: also fsk_demod's complex AGC output)
    DevBuf<float> d_atan_tab;
    long last_pm = 0;                    // samples through the carrier PLL in the last batch
    float snr_now = 0.f, snr_peak = 0.f; // M2M4SNREstimator::snr() after the last push / its maximum so far (module_psk_demod.cpp:190-194)
    long max_batch;
    // fsk_demod: quadrature demodulator, float DC blocker and AGC outputs (agc2_out with a 32-sample front pad: the FIR's history)
    bool fsk = false;
    DevBuf<float> quad_out, dc2_out, agc2_out;
    // complex AGC output (pm_agc) -> k_quad -> k_fsk_dc -> k_fsk_agc -> k_fir_real -> the clock recovery's input in bufA
    void stage_fsk(long n, const FirTaps &taps, int cur, int nxt);
    int slot_cap_for(int L) const;
    int choose_L(long n) const;
};

void design_rrc(double gain, double fs, double rs, double alpha, int ntaps, std::vector<float> &out);
void design_mm_bank(std::vector<float> &out);
// RationalResamplerBlock::set_ratio's bank for the reduced (I, D): returns taps per arm, bank[arm * ntaps + k]
int design_resampler_bank(unsigned I, unsigned D, std::vector<float> &bank);

} // namespace b200
