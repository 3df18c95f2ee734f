// C ABI + host driver of the demodulator (see include/b200dsp.h, demod_host.h).
#define B200_DEFINE_KERNELS
#include "demod_host.h"
#include "power_decim_taps.inc"
#include <string>
#include <algorithm>
#include <cmath>
#include <mutex>
#include <type_traits>

namespace b200
{
static thread_local std::string g_err;
void set_error(const char *fmt, ...)
{
    char b[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(b, sizeof(b), fmt, ap);
    va_end(ap);
    g_err = b;
}
const char *last_error_cstr() { return g_err.c_str(); }

void check_device(int device)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        throw ApiError(B200_ENODEV, std::string("no CUDA device: ") + cudaGetErrorString(e) + " (this library has no CPU fallback)");
    if (device < 0 || device >= n)
        throw ApiError(B200_ENODEV, "CUDA device ordinal out of range");
    cudaDeviceProp p;
    B200_CUDA(cudaGetDeviceProperties(&p, device));
    if (p.major != 9 || p.minor != 0)
        throw ApiError(B200_ENODEV, std::string("device ") + p.name + " is not sm_90: the kernels are built for sm_90a only");
}

// Root-raised-cosine design, double precision, odd length, normalised to unit DC gain.
// Formula and evaluation order follow firdes::root_raised_cosine (src-core/common/dsp/filter/firdes.cpp:34-78) so the
// float taps come out identical.
void design_rrc(double gain, double fs, double rs, double alpha, int ntaps, std::vector<float> &out)
{
    ntaps |= 1;
    out.assign(ntaps, 0.f);
    const double spb = fs / rs;
    double sum = 0;
    for (int i = 0; i < ntaps; i++) {
        const double xi = i - ntaps / 2;
        double x1 = M_PI * xi / spb, x2 = 4 * alpha * xi / spb, x3 = x2 * x2 - 1;
        double num, den;
        if (fabs(x3) >= 0.000001) {
            num = (i != ntaps / 2) ? cos((1 + alpha) * x1) + sin((1 - alpha) * x1) / (4 * alpha * xi / spb)
                                   : cos((1 + alpha) * x1) + (1 - alpha) * M_PI / (4 * alpha);
            den = x3 * M_PI;
        } else {
            if (alpha == 1) {
                out[i] = -1;
                sum += out[i];
                continue;
            }
            x3 = (1 - alpha) * x1;
            x2 = (1 + alpha) * x1;
            num = (sin(x2) * (1 + alpha) * M_PI - cos(x3) * ((1 - alpha) * M_PI * spb) / (4 * alpha * xi) + sin(x3) * spb * spb / (4 * alpha * xi * xi));
            den = -32 * M_PI * alpha * alpha * xi / spb;
        }
        out[i] = (float)(4 * alpha * num / den);
        sum += out[i];
    }
    for (int i = 0; i < ntaps; i++)
        out[i] = (float)(out[i] * gain / sum);
}

// 128-arm x 8-tap polyphase interpolator of the M&M block: Nuttall-windowed sinc prototype of 1024 taps
// (src-core/common/dsp/window/window.cpp:9-50), arm a / tap k = prototype[(127-a) + 128k] (polyphase_bank.cpp:35-36).
void design_mm_bank(std::vector<float> &out)
{
    const int arms = 128, per = 8, count = arms * per;
    out.assign(count, 0.f);
    const double w[4] = {0.355768, 0.487396, 0.144232, 0.012604};
    const double omega = 2.0 * M_PI * ((0.5 / (double)arms) / 1.0), half = count / 2.0, corr = arms * omega / M_PI;
    for (int i = 0; i < count; i++) {
        const double t = (double)i - half + 0.5, x = t * omega;
        const double sinc = (x == 0.0) ? 1.0 : sin(x) / x;
        double win = 0, sign = 1;
        for (int c = 0; c < 4; c++) {
            win += sign * w[c] * cos((double)c * 2.0 * M_PI * (t - half) / count);
            sign = -sign;
        }
        out[((arms - 1) - (i % arms)) * per + i / arms] = (float)(sinc * win * corr);
    }
}

// Kaiser-windowed low-pass of the rational resampler, evaluated like firdes::design_resampler_filter_float -> firdes::low_pass ->
// window::kaiser (src-core/common/dsp/filter/firdes.cpp:276-301, 80-120, 453-478, Izero 357-373) so the float taps come out
// identical, then folded into arms like PolyphaseBank::init (resamp/polyphase_bank.cpp:6-39).
static double izero(double x)
{
    double sum = 1, u = 1;
    int n = 1;
    const double halfx = x / 2.0;
    do {
        double temp = halfx / (double)n;
        n += 1;
        temp *= temp;
        u *= temp;
        sum += u;
    } while (u >= 1E-21 * sum);
    return sum;
}

int design_resampler_bank(unsigned I, unsigned D, std::vector<float> &bank)
{
    const float beta = 7.0f, halfband = 0.5f, fractional_bw = 0.4f, rate = (float)I / (float)D;
    float trans_width, mid;
    if (rate >= 1.0f) {
        trans_width = halfband - fractional_bw;
        mid = (float)(halfband - trans_width / 2.0);
    } else {
        trans_width = rate * (halfband - fractional_bw);
        mid = (float)(rate * halfband - trans_width / 2.0);
    }
    double gain = I;
    const double fs = I, cutoff = mid, tw = trans_width, b = beta;
    const double a = b / 0.1102 + 8.7;
    int ntaps = (int)(a * fs / (22.0 * tw));
    if ((ntaps & 1) == 0)
        ntaps++;
    std::vector<float> taps(ntaps), w(ntaps);
    {
        const double IBeta = 1.0 / izero(b), inm1 = 1.0 / ((double)(ntaps - 1));
        w[0] = (float)IBeta;
        for (int i = 1; i < ntaps - 1; i++) {
            const double temp = 2 * i * inm1 - 1;
            w[i] = (float)(izero(b * sqrt(1.0 - temp * temp)) * IBeta);
        }
        w[ntaps - 1] = (float)IBeta;
    }
    const int M = (ntaps - 1) / 2;
    const double fwT0 = 2 * M_PI * cutoff / fs;
    for (int n = -M; n <= M; n++)
        taps[n + M] = n == 0 ? (float)(fwT0 / M_PI * w[n + M]) : (float)(sin(n * fwT0) / (n * M_PI) * w[n + M]);
    double fmax = taps[M];
    for (int n = 1; n <= M; n++)
        fmax += 2 * taps[n + M];
    gain /= fmax;
    for (int i = 0; i < ntaps; i++)
        taps[i] = (float)(taps[i] * gain);
    int nt = (ntaps + (int)I - 1) / (int)I;
    if (fmod((double)ntaps / (double)I, 1.0) > 0.0)
        nt++;
    bank.assign((size_t)I * nt, 0.f);
    for (int i = 0; i < (int)I * nt; i++)
        bank[(size_t)((I - 1) - (i % I)) * nt + i / I] = i < ntaps ? taps[i] : 0.f;
    return nt;
}

static unsigned gcd_u(unsigned a, unsigned b)
{
    while (b) {
        unsigned t = a % b;
        a = b;
        b = t;
    }
    return a;
}

// SmartResamplerBlock(input, final_samplerate, samplerate) -> (unsigned interpolation, unsigned decimation), smart_resampler.cpp:8-61:
// a power-of-two decimator by 1 << decim_power first when the input rate is at least twice the final one (power_decim.cpp:13-29),
// then the rational resampler by the reduced I / D behind it, unless the decimator alone reached the final rate (rational = false)
struct SmartRatio
{
    int decim_power;
    bool rational;
    unsigned I, D;
};
static SmartRatio smart_resampler_ratio(unsigned interpolation, unsigned decimation)
{
    SmartRatio r{0, true, 0, 0};
    double rsamp_in = decimation, fout = interpolation;
    if (decimation > interpolation) {
        const int best_power = (int)floor(log2((double)(decimation / interpolation))); // (unsigned division, as the reference)
        if (best_power > 0) {
            r.decim_power = std::min(best_power, PD_NPLANS);
            rsamp_in = (double)decimation / (double)(1 << r.decim_power);
        }
        r.rational = rsamp_in != fout;
        double t; // "ensure it's all integer" (smart_resampler.cpp:35-40)
        while (modf(rsamp_in, &t) != 0 || modf(fout, &t) != 0) {
            rsamp_in *= 10;
            fout *= 10;
        }
    }
    const unsigned g = gcd_u((unsigned)fout, (unsigned)rsamp_in);
    r.I = (unsigned)fout / g;
    r.D = (unsigned)rsamp_in / g;
    return r;
}

// the working window of samples per symbol of the loops (module_psk_demod.cpp:65-70); min_sps / max_sps > 0 replace its ends
struct SpsWindow
{
    float lo, hi;
};
static SpsWindow sps_window(int constellation, float min_sps = 0, float max_sps = 0)
{
    SpsWindow w{constellation == B200_OQPSK ? 1.6f : 1.1f, constellation == B200_OQPSK ? 2.4f : 4.0f};
    if (min_sps > 0)
        w.lo = min_sps;
    if (max_sps > 0)
        w.hi = max_sps;
    return w;
}

// Calls f(std::integral_constant<int, F>{}) with F the kernels' template index (0 cf32, 1 cs16, 2 cs8) of the sample format fmt.
template <class Fn> static auto with_fmt(int fmt, Fn &&f)
{
    if (fmt == B200_CF32)
        return f(std::integral_constant<int, 0>{});
    if (fmt == B200_CS16)
        return f(std::integral_constant<int, 1>{});
    return f(std::integral_constant<int, 2>{});
}
static int fmt_bytes(int fmt)
{
    return with_fmt(fmt, [](auto F) { return RawBytes<F>::v; });
}

static int round_up16(double v) { return ((int)std::ceil(v / 16.0)) * 16; }
// k_mm instantiation: STRICT (test hook), GARDNER (clock_recovery 1), FIX (the input still needs its rotation / OQPSK delay), REAL
// (fsk_demod: MMClockRecoveryBlock<float>'s detector on the real part; no Gardner, no fix-up)
static decltype(&k_mm<false, false, false>) mm_kernel(bool strict, bool gardner, bool fix, bool real = false)
{
    if (real)
        return strict ? k_mm<true, false, false, true> : k_mm<false, false, false, true>;
    if (strict)
        return gardner ? (fix ? k_mm<true, true, true> : k_mm<true, true, false>) : (fix ? k_mm<true, false, true> : k_mm<true, false, false>);
    return gardner ? (fix ? k_mm<false, true, true> : k_mm<false, true, false>) : (fix ? k_mm<false, false, true> : k_mm<false, false, false>);
}
// a run of r consecutive unconverged junctions needs r rounds; idle rounds cost two empty launches
constexpr int REPAIR_ROUNDS = 8;

Demod::Demod(const b200_demod_cfg &c) : cfg(c)
{
    B200_REQUIRE(c.samplerate > 0 && c.symbolrate > 0, B200_EINVAL, "samplerate / symbolrate must be present and positive");
    B200_REQUIRE(c.constellation >= B200_BPSK && c.constellation <= B200_NONE, B200_EINVAL, "unknown constellation %d", c.constellation);
    B200_REQUIRE(c.format >= B200_CF32 && c.format <= B200_CS8, B200_EINVAL, "unsupported baseband_format %d (cf32/cs16/cs8 only)", c.format);
    B200_REQUIRE((c.rrc_taps | 1) == FIR_NT, B200_EINVAL, "rrc_taps=%d: only the 31-tap RRC kernel is built", c.rrc_taps);
    B200_REQUIRE(c.max_batch >= 4096, B200_EINVAL, "max_batch must be >= 4096 samples");
    B200_REQUIRE(c.agc_rate > 0 && c.agc_rate < 0.5f, B200_EINVAL, "agc_rate out of range");
    B200_REQUIRE(c.clock_gain_mu > 0 && (c.fsk_demod || c.pll_bw > 0), B200_EINVAL, "loop gains must be positive");
    B200_REQUIRE(c.clock_recovery == 0 || c.clock_recovery == 1, B200_EINVAL, "clock_recovery must be 0 (M&M) or 1 (Gardner)");
    const long fs = (long)c.samplerate, rs = (long)c.symbolrate;
    const float final_fs = c.final_samplerate > 0 ? (float)c.final_samplerate : (float)fs; // float final_samplerate (module_demod_base.h:67)
    sps = final_fs / (float)rs;
    // the loops are built for the reference's working window (module_demod_base.h:71-72, module_psk_demod.cpp:65-70); outside it
    // the reference resamples first: pass final_samplerate = b200_demod_final_samplerate(...)
    pm = c.pm_demod != 0;
    pm_after = pm && c.pm_resample_after_pll != 0;
    if (pm) {
        // PMDemodModule (module_pm_demod.cpp:12-88): BPSK behind a carrier PLL; its Costas loop is order 2 with the default frequency limit
        B200_REQUIRE(c.constellation == B200_BPSK, B200_EINVAL, "pm_demod recovers BPSK: constellation must be bpsk");
        B200_REQUIRE(c.pm_pll_bw > 0 && c.pm_pll_bw < 0.5f && c.pm_pll_max_offset > 0, B200_EINVAL, "pm_demod: pll_bw / pll_max_offset out of range");
        B200_REQUIRE(!c.post_costas_dc && c.clock_recovery == 0, B200_EINVAL, "pm_demod has no post-Costas DC blocker and uses the M&M clock recovery");
        cfg.costas_max_offset = 1.0f; // CostasLoopBlock(rrc->output_stream, d_loop_bw, 2): freq_limit defaults to 1.0 (costas_loop.h:27)
    }
    if (c.has_carrier) { // module_psk_demod.cpp:93-113
        B200_REQUIRE(!pm, B200_EINVAL, "has_carrier is psk_demod's carrier mode, not pm_demod's");
        B200_REQUIRE(c.constellation == B200_BPSK, B200_EINVAL, "For carrier mode, constellation must be BPSK!");
        B200_REQUIRE(c.carrier_pll_bw > 0 && c.carrier_pll_bw < 0.5f && c.carrier_pll_max_offset > 0, B200_EINVAL, "carrier_pll_bw / carrier_pll_max_offset out of range");
    }
    fsk = c.fsk_demod != 0;
    if (fsk) { // FSKDemodModule (module_fsk_demod.cpp:13-84): no Costas loop, the real M&M; the base working window (module_demod_base.h:71-72)
        B200_REQUIRE(c.constellation == B200_BPSK, B200_EINVAL, "fsk_demod gives one real symbol per sample pair: constellation must be bpsk");
        B200_REQUIRE(!pm, B200_EINVAL, "fsk_demod cannot be combined with pm_demod");
        B200_REQUIRE(!c.has_carrier, B200_EINVAL, "fsk_demod cannot be combined with has_carrier");
        B200_REQUIRE(!c.post_costas_dc, B200_EINVAL, "fsk_demod cannot be combined with post_costas_dc");
        B200_REQUIRE(c.clock_recovery == 0, B200_EINVAL, "fsk_demod uses the M&M clock recovery (clock_recovery Gardner is psk_demod's)");
    }
    SpsWindow win = sps_window(c.constellation);
    if (pm) // MAX_SPS = 10 for pm_demod ("we do NOT want to resample unless really necessary", module_pm_demod.cpp:56)
        win.hi = 10.0f;
    B200_REQUIRE(sps >= win.lo * 0.999f && sps <= win.hi * 1.001f, B200_EINVAL,
                 "samples per symbol %.4f outside [%.1f, %.1f]: set final_samplerate (b200_demod_final_samplerate) so that the front-end resampler runs", sps,
                 win.lo, win.hi);
    if (c.final_samplerate > 0 && (long)c.final_samplerate != fs && c.front_resample != 2) {
        const unsigned interpolation = (unsigned)final_fs, decimation = (unsigned)fs;
        B200_REQUIRE(interpolation > 0, B200_EINVAL, "final_samplerate too small");
        const SmartRatio r = smart_resampler_ratio(interpolation, decimation);
        if (r.decim_power > 0) {
            const PdPlan &plan = PD_PLANS[r.decim_power - 1];
            for (int i = 0; i < plan.nstages; i++) {
                DecimStage st;
                st.D = plan.stages[i].decimation;
                st.nt = plan.stages[i].ntaps;
                st.taps_rev.resize(st.nt);
                for (int k = 0; k < st.nt; k++)
                    st.taps_rev[k] = PD_TAPS[plan.stages[i].offset + st.nt - 1 - k]; // decimating_fir.cpp:30: reversed
                decim.push_back(std::move(st));
            }
            decim_total = 1 << r.decim_power;
        }
        if (r.rational) {
            rs_I = (int)r.I;
            rs_D = (int)r.D;
            rs_nt = design_resampler_bank(r.I, r.D, rs_bank);
            B200_REQUIRE(rs_nt <= RS_MAX_TAPS, B200_EUNSUPPORTED, "resampler arm of %d taps exceeds the built maximum %d", rs_nt, RS_MAX_TAPS);
            resamp = true;
        } else if (c.iq_swap && decim.empty() && !pm_after) {
            rs_bank.assign(1, 1.0f);
            resamp = true;
        }
    } else if (c.iq_swap && !pm_after) { // the plain swap runs as the identity resampler
        rs_bank.assign(1, 1.0f);
        resamp = true;
    }
    check_device(c.device);
    DeviceGuard g(c.device);
    bps = c.constellation == B200_BPSK ? 1 : 2;
    {
        // phasor steps of the two rotators as fractions of a turn (0.64 fixed point): the angle of the FLOAT pair (cos, sin)(2 pi f / fs)
        // the reference multiplies by (freq_shift.cpp:44-45, pm_to_bpsk.cpp:12)
        auto turn_step = [](double freq, double rate) -> unsigned long long {
            const double w = 2.0 * M_PI * (freq / rate); // hz_to_rad (common/dsp/block.cpp:17)
            const float ir = (float)cos(w), ii = (float)sin(w);
            long double a = atan2l((long double)ii, (long double)ir) / (2.0L * 3.14159265358979323846264338327950288L);
            if (a < 0)
                a += 1.0L;
            const long double v = a * 18446744073709551616.0L;
            return v >= 18446744073709551615.0L ? 0ull : (unsigned long long)v;
        };
        if (pm) {
            // PMToBPSK(pll out, d_resample_after_pll ? d_samplerate : final_samplerate, subcarrier_offset == 0 ? d_symbolrate : subcarrier_offset),
            // float arguments, shifting DOWN by that frequency (module_pm_demod.cpp:67, pm_to_bpsk.cpp:10-13)
            const float rate = pm_after ? (float)fs : final_fs;
            const unsigned long sub = (unsigned long)c.pm_subcarrier_offset;
            const float f = sub == 0 ? (float)rs : (float)sub;
            pm_dturn = turn_step(-(double)f, (double)rate);
        }
        if (c.freq_shift != 0) // FreqShiftBlock(input, d_samplerate, d_frequency_shift): long parameters (module_demod_base.h:56, .cpp:122-123)
            fs_dturn = turn_step((double)(long)c.freq_shift, (double)fs);
    }
    order = fsk ? 0 : (c.constellation == B200_BPSK ? 2 : (c.constellation == B200_8PSK ? 8 : (c.constellation == B200_NONE ? 0 : 4)));
    max_batch = c.max_batch;
    max_work = resamp ? std::max<long>(max_batch, (long)((double)max_batch * rs_I / rs_D) + 64) : max_batch; // (a decimator in front only shrinks it)
    if (pm || c.has_carrier) {
        // carrier PLL warm-up: the loop is linear (its detector is the input's own phase minus the loop phase), two copies approach each
        // other like exp(-n * bw * 1.5): 24 / bw samples bring any start state below float resolution of the phase
        Wp = round_up16(24.0 / (pm ? c.pm_pll_bw : c.carrier_pll_bw));
    }
    design_rrc(1, final_fs, (double)(int)rs, c.rrc_alpha, c.rrc_taps, rrc);
    design_mm_bank(bank);
    // Costas warm-up: 24 loop time constants for orders 2/4; the order-8 detector has about a third of the gain (measured on the
    // psk8 signal: 0.94 % of the samples off by >1e-5 with 24/bw, 0.10 % with 48/bw, 0.015 % with 96/bw)
    Wc = round_up16((c.constellation == B200_8PSK ? 72.0 : 24.0) / c.pll_bw);
    // M&M warm-up: the timing loop has to land on the sequential trajectory to ~1e-4 sample. Its time constant is 1/(gain_mu * K)
    // symbols with a TED gain K that falls with the samples per symbol (the pulse slope per sample) and is about half as large for
    // BPSK (one rail), i.e. ~ sps^2 in samples. Measured on 2^21-sample signals: QPSK sps 2.57 with 70/gain_mu samples sits at the
    // reference's own chaos floor (1.1-1.6 % of the symbols off by an interpolator arm); BPSK needs 240/gain_mu at sps 2.5 and
    // 4x that... i.e. (sps/2.5)^2 more at sps 3.6 (0.5 % = floor; with half of it 3 %, with a quarter 49 %).
    {
        const double ref_sps = c.constellation == B200_BPSK ? 2.5 : 2.5714;
        const double scale = std::max(1.0, (double)sps * sps / (ref_sps * ref_sps));
        // QPSK-type: 70/gain_mu left the segments a median 1.1e-4 sample off the sequential trajectory at their first owned symbol
        // (1.6 % of the symbols of 1024-sample segments off by an interpolator arm, against 0.3-0.4 % for the reference perturbed by
        // 1e-6: tests/floors.py); the error falls by e per ~1200 samples: 87.5/gain_mu -> 4e-5 (0.7 %)
        Wm = round_up16((c.constellation == B200_BPSK ? 240.0 : 87.5) * scale / c.clock_gain_mu);
    }
    // gear shift (k_costas / k_mm): the first quarter of a warm-up runs first order at 4x the gain
    Gc = (Wc / 4) & ~15;
    Gm = (Wm / 4) & ~15;
    // junction tolerances (a junction outside them is repaired = re-run as the exact sequential continuation). Orders 2 / 4 on
    // non-offset signals: converged segments sit within 6e-6 rad of their predecessor (float rounding noise of two loops on the same
    // trajectory), so 1e-5 only catches real stragglers and bounds the output error of a junction to ~1e-5 |v|. The OQPSK / 8PSK
    // detectors leave 0.1-0.4 % of the warm-ups ~1e-3 off (hang-ups near the unstable lock point); a junction that far off seeds
    // sign-decision events in the segment (a 7e-3 rad kick each), hence 2e-5 there too.
    if (order == 2 || (order == 4 && c.constellation != B200_OQPSK)) {
        tol_cphase = 1e-5f;
        tol_cfreq = 2e-6f;
    } else if (order) { // repairs are common here (1-4 % of the junctions): a round costs about half a k_costas pass
        tol_cphase = 2e-5f;
        tol_cfreq = 4e-6f;
    }
    tol_mm = 0.01f; // samples (1.3 interpolator arms)
    // a timing error moves omega by gain_omega and mu by gain_mu per unit of the detector's output: the same disagreement, in omega
    tol_momega = tol_mm * c.clock_gain_omega / c.clock_gain_mu;
    int dev_sms = 132;
    cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, c.device);
    seg_cap_threads = dev_sms * 2 * SEG_THREADS; // the segment count aims at 2 resident CTAs of the loop kernels per SM
    {
        // in a pipelined chain the demodulator of batch i runs next to the decoder of batch i-1 and is the longer of the two: its
        // kernels take freed SM slots first
        int lo = 0, hi = 0;
        B200_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        B200_CUDA(cudaStreamCreateWithPriority(&stream, cudaStreamNonBlocking, hi));
    }
    for (auto &e : ev)
        B200_CUDA(cudaEventCreate(&e));
    raw.alloc((size_t)max_batch * fmt_bytes(c.format) + 64);
    B200_CUDA(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
    for (auto &p : pf)
        B200_CUDA(cudaEventCreateWithFlags(&p.done, cudaEventDisableTiming));
    bufA.alloc(max_work + 64);
    bufB.alloc(max_work + 64);
    if (c.keep_stages) {
        agc_dump.alloc(max_work);
        fir_dump.alloc(max_work);
    }
    const int ntiles_max = (int)((max_work + FIR_TILE - 1) / FIR_TILE);
    tile_map.alloc(ntiles_max + 1);
    tile_map3.alloc(ntiles_max + 1);
    seeds.alloc(ntiles_max + 2);
    agc_need.alloc(2);
    agc_need.zero(stream);
    {
        // one wave of resident warps, each owning a range of tiles (k_agc_fir_w: 4 independent warps per CTA, 11.5 KB of smem)
        int per_sm = 0;
        const int agc_fmt = (resamp || c.dc_block || !decim.empty()) ? B200_CF32 : c.format;
        with_fmt(agc_fmt, [&](auto F) {
            B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_agc_fir_w<F, false, false>, 32 * FW_WARPS, 0));
        });
        fir_ctas = std::max(1, per_sm) * dev_sms;
        fir_warps = fir_ctas * FW_WARPS;
        if (const char *e = getenv("B200_AGC_WARM_TILES")) // 0 forces the exact (scanned-seed) pass: test hook
            agc_warm_max = std::max(0, atoi(e));
    }
    // worst-case segment count / slot storage: 4096 <= L <= 16384 (choose_L), nseg * cap(L) <= n/omin + L/omin + 16 (nseg + 1)
    const int lmin = 4096;
    const long nseg_max = (max_work + lmin - 1) / lmin + 1;
    crec.alloc(nseg_max);
    mrec.alloc(nseg_max);
    // nseg * ckpt_per_seg(L) < (n + L) / CKPT; a SEQUENTIAL debug run has one segment of n samples
    cck.alloc((max_work + 16384) / CKPT + 1);
    mck.alloc((max_work + 16384) / CKPT + 1);
    quad.alloc(nseg_max);
    offs.alloc(nseg_max + 1);
    repair.alloc(1025);
    const double omin = sps * (1.0 - c.clock_omega_limit) - 0.01;
    slots.alloc((size_t)(max_work / omin) + (size_t)(16384 / omin) + nseg_max * 24 + 1024);
    sym_out.alloc((size_t)(max_work / omin) + 1024);
    soft.alloc(((size_t)(max_work / omin) + 1024) * bps);
    d_bank.alloc(128 * 8);
    if (cfg.dc_block || cfg.post_costas_dc || cfg.has_carrier) {
        const int nt = (int)((std::max(max_batch, max_work) + FIR_TILE - 1) / FIR_TILE);
        dc_map.alloc(nt + 1);
        dc_seeds.alloc(nt + 2);
    }
    if (cfg.dc_block)
        dc_out.alloc(max_batch + 64);
    if (cfg.freq_shift != 0)
        fs_out.alloc(max_batch + 64);
    if (pm || cfg.has_carrier) {
        const long npm = std::max(max_batch, max_work) + 64;
        if (pm) {
            pm_agc.alloc(npm);
            pm_out.alloc(npm);
        }
        pm_pll.alloc(npm);
        // fast_atan2f's table (fast_trig.cpp:16-61): the arctangent of k / 255 through seven significant digits, entry 256 = entry 255
        std::vector<float> tab(260, 0.f);
        char buf[40];
        for (int k = 0; k < 256; k++) {
            snprintf(buf, sizeof buf, "%.6e", atan((double)k / 255.0));
            tab[k] = (float)strtod(buf, nullptr);
        }
        tab[256] = tab[255];
        d_atan_tab.alloc(260);
        B200_CUDA(cudaMemcpyAsync(d_atan_tab.p, tab.data(), 260 * sizeof(float), cudaMemcpyHostToDevice, stream));
        B200_CUDA(cudaStreamSynchronize(stream)); // (tab is a local)
        B200_CUDA(cudaFuncSetAttribute(k_pll, cudaFuncAttributeMaxDynamicSharedMemorySize, PLL_SMEM_BYTES));
    }
    if (fsk) {
        pm_agc.alloc(max_work + 64);
        quad_out.alloc(max_work + 64);
        dc2_out.alloc(max_work + 64);
        agc2_out.alloc(max_work + 64 + 32);
    }
    if (cfg.post_costas_dc) {
        B200_REQUIRE(order != 0 && c.constellation != B200_OQPSK, B200_EINVAL, "post_costas_dc needs a Costas loop and is not built for OQPSK");
        pdc_out.alloc(max_work + 64);
        pdc_out.zero(stream);
    }
    {
        long cap = max_batch;
        for (auto &stg : decim) {
            cap = cap / stg.D + 2;
            stg.d_taps.alloc(stg.nt);
            stg.tail[0].alloc(stg.nt);
            stg.tail[1].alloc(stg.nt);
            stg.tail[0].zero(stream);
            stg.tail[1].zero(stream);
            stg.out.alloc(cap + 64);
            B200_CUDA(cudaMemcpyAsync(stg.d_taps.p, stg.taps_rev.data(), stg.nt * sizeof(float), cudaMemcpyHostToDevice, stream));
        }
    }
    if (resamp) {
        d_rs_bank.alloc(rs_bank.size());
        rs_out.alloc(max_work + 64);
        B200_CUDA(cudaMemcpyAsync(d_rs_bank.p, rs_bank.data(), rs_bank.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
    }
    st.alloc(1);
    B200_CUDA(cudaMemcpyAsync(d_bank.p, bank.data(), 128 * 8 * sizeof(float), cudaMemcpyHostToDevice, stream));
    h_total.alloc(1);
    h_state.alloc(1);
    init_state();
    bufA.zero(stream);
    bufB.zero(stream);
    for (int v = 0; v < 10; v++)
        B200_CUDA(cudaFuncSetAttribute(mm_kernel(v & 1, v & 2, v & 4, v >= 8), cudaFuncAttributeMaxDynamicSharedMemorySize, MM_SMEM_BYTES));
    B200_CUDA(cudaFuncSetAttribute(k_costas<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, COSTAS_SMEM_BYTES));
    B200_CUDA(cudaFuncSetAttribute(k_costas<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, COSTAS_SMEM_BYTES));
    B200_CUDA(cudaFuncSetAttribute(k_costas<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, COSTAS_SMEM_BYTES));
    B200_CUDA(cudaStreamSynchronize(stream));
}

Demod::~Demod()
{
    DeviceGuard g(cfg.device);
    if (stream)
        cudaStreamSynchronize(stream);
    for (auto &e : ev)
        cudaEventDestroy(e);
    if (copy_stream) {
        cudaStreamSynchronize(copy_stream);
        cudaStreamDestroy(copy_stream);
    }
    for (auto &p : pf)
        if (p.done)
            cudaEventDestroy(p.done);
    if (stream)
        cudaStreamDestroy(stream);
}

// initial loop state, uploaded on the stream: AGC gain 1 (module_demod_base.cpp:207), Costas 0/0, M&M mu / omega (clock_recovery_mm.cpp:11)
void Demod::init_state()
{
    memset(h_state.p, 0, sizeof(DemodDevState));
    h_state.p->gain[0] = h_state.p->gain[1] = 1.0f;
    h_state.p->gain2[0] = h_state.p->gain2[1] = 1.0f;
    h_state.p->fgain[0] = h_state.p->fgain[1] = 1.0f; // AGCBlock<float>(.., 0.1, 0.5, 1.0, 65535): gain 1 (module_fsk_demod.cpp:70)
    for (int i = 0; i < 2; i++) {
        h_state.p->mm[i].mu = cfg.clock_mu;
        h_state.p->mm[i].omega = sps;
    }
    B200_CUDA(cudaMemcpyAsync(st.p, h_state.p, sizeof(DemodDevState), cudaMemcpyHostToDevice, stream));
}

void Demod::reset()
{
    DeviceGuard g(cfg.device);
    B200_CUDA(cudaStreamSynchronize(stream));
    init_state();
    pm_pos = fs_pos = 0;
    B200_CUDA(cudaStreamSynchronize(stream));
    parity = 0;
    last_n = last_syms = 0;
    rs_inc = rs_ctr = 0;
    for (auto &stg : decim) {
        stg.inc = 0;
        stg.tail[0].zero(stream);
        stg.tail[1].zero(stream);
    }
    B200_CUDA(cudaStreamSynchronize(stream));
}

int Demod::choose_L(long n) const
{
    // one segment per thread; aim at one full wave of resident threads, but keep segments within [4096, 16384] samples: a segment
    // shorter than a few loop time constants (M&M: ~1200 samples) spends its whole life in the tail of its warm-up transient
    if (dbg_seg_len > 0)
        return dbg_seg_len;
    long L = (n + seg_cap_threads - 1) / seg_cap_threads;
    L = std::max<long>(4096, std::min<long>(16384, L));
    return (int)((L + 15) / 16 * 16);
}

int Demod::slot_cap_for(int L) const
{
    const double omin = sps * (1.0 - cfg.clock_omega_limit) - 0.01;
    return (int)(L / omin) + 16;
}

template <int FMT> static void launch_front(Demod &d, const void *raw, long n, int ntiles, FirTaps taps, const AgcUnit &u)
{
    DemodDevState *S = d.st.p;
    // one wave of resident warps, each running a range of R consecutive tiles. Any R >= 1 computes the same stream; the floor of 4
    // amortises the walk back that proves a range's start gain (normally 4-5 tiles of map-only work)
    const int R = d.dbg_range_tiles > 0 ? d.dbg_range_tiles : std::max(4, (ntiles + d.fir_warps - 1) / d.fir_warps);
    d.last_R = R;
    const int nranges = (ntiles + R - 1) / R;
    const int grid = (nranges + FW_WARPS - 1) / FW_WARPS;
    AgcCtl ctl;
    ctl.seeds = d.seeds.p;
    ctl.need = d.agc_need.p;
    ctl.epoch = ++d.agc_epoch;
    ctl.warm_max = d.agc_warm_max;
    ctl.max_gain = u.max_gain;
    const int *need = d.agc_need.p + (ctl.epoch & 1);
    const auto fir = u.dump ? k_agc_fir_w<FMT, true, false> : k_agc_fir_w<FMT, false, false>;
    for (int pass = 0; pass < 2; pass++) {
        ctl.seeded = pass;
        if (pass) { // exact pass: returns at once unless the fast pass asked for it
            k_agc_compose<FMT><<<std::min(ntiles, d.fir_ctas * 2), FIR_THREADS, 0, d.stream>>>(raw, n, u.rate, u.max_gain, need, ~0, ntiles, d.tile_map.p);
            k_tile_scan<<<1, 1024, 0, d.stream>>>(d.tile_map.p, ntiles, u.gain_in, need, ~0, d.seeds.p, &S->agc_exact);
        }
        fir<<<grid, 32 * FW_WARPS, 0, d.stream>>>(raw, n, u.rate, u.gain_in, R, ctl, taps, u.tail_in, u.tail_out, u.fir_out, u.dump, u.gain_out, &S->flags);
    }
    // clamp pass: the gain reached max_gain somewhere in this batch (silent input), so the unclamped maps above do not describe
    // the reference's loop; redo the stage with the clamped ones. All three launches return at once otherwise.
    ctl.seeded = 1;
    k_agc_compose<FMT><<<std::min(ntiles, d.fir_ctas * 2), FIR_THREADS, 0, d.stream>>>(raw, n, u.rate, u.max_gain, &S->flags, 1, ntiles, d.tile_map3.p);
    k_tile_scan<<<1, 1024, 0, d.stream>>>(d.tile_map3.p, ntiles, u.gain_in, &S->flags, 1, d.seeds.p, nullptr);
    const auto fir_clamp = u.dump ? k_agc_fir_w<FMT, true, true> : k_agc_fir_w<FMT, false, true>;
    fir_clamp<<<grid, 32 * FW_WARPS, 0, d.stream>>>(raw, n, u.rate, u.gain_in, R, ctl, taps, u.tail_in, u.tail_out, u.fir_out, u.dump, u.gain_out, &S->flags);
    d.launches += 7;
}
static void launch_front_fmt(Demod &d, int fmt, const void *raw, long n, FirTaps taps, const AgcUnit &u)
{
    const int ntiles = (int)((n + FIR_TILE - 1) / FIR_TILE);
    with_fmt(fmt, [&](auto F) { launch_front<F>(d, raw, n, ntiles, taps, u); });
}

// FreqShiftBlock / PMToBPSK: see k_rotator. pos = samples the rotator has seen before this batch.
void Demod::run_rotator(const void *src, int fmt, long n, int iq_swap, int imag_only, unsigned long long dturn, unsigned long long pos, float2 *dst)
{
    const unsigned grid = (unsigned)((n + 8 * 256 - 1) / (8 * 256));
    const unsigned long long turn0 = pos * dturn; // mod 2^64 = mod one turn
    with_fmt(fmt, [&](auto F) { k_rotator<F><<<grid, 256, 0, stream>>>(src, n, iq_swap, imag_only, turn0, dturn, dst); });
    launches++;
}

// CorrectIQBlock (utils/correct_iq.cpp:18-35, alpha correct_iq.h:24) over n samples at src: per-tile maps, their scan from the carried
// accumulator acc_in, then the output and the accumulator after the batch (acc_out)
void Demod::run_dc(const void *src, int fmt, int iq_swap, long n, const float2 *acc_in, float2 *acc_out, float2 *dst)
{
    const int nt = (int)((n + FIR_TILE - 1) / FIR_TILE);
    const float alpha = 0.0001f, beta = 1.0f - alpha;
    with_fmt(fmt, [&](auto F) {
        k_dc_tile<F><<<nt, FIR_THREADS, 0, stream>>>(src, n, iq_swap, alpha, beta, dc_map.p);
        k_tile_scan<<<1, 1024, 0, stream>>>(dc_map.p, nt, acc_in, nullptr, 0, dc_seeds.p, nullptr);
        k_dc_apply<F><<<nt, FIR_THREADS, 0, stream>>>(src, n, iq_swap, alpha, beta, dc_seeds.p, dst, acc_out);
    });
    launches += 3;
}

// A loop stage: round(grid, repair_list, repair_count, r) launches the loop kernel and its junction check. Round 0 runs all segments,
// rounds 1..REPAIR_ROUNDS re-run the flagged ones on 8 CTAs (both kernels return at once when no junction is flagged).
template <class Round> static void run_loop_stage(Demod &d, int nblk, Round round)
{
    round(nblk, nullptr, nullptr, 0);
    for (int r = 1; r <= REPAIR_ROUNDS; r++)
        round(8, d.repair.p + 1, d.repair.p, r);
    d.launches += 2 + 2 * REPAIR_ROUNDS;
}

// pm_demod: PLLCarrierTrackingBlock over the AGC output (pm_agc -> pm_pll; junction check / repair rounds as for the Costas loop, with
// order 1: the lock point is unique), then PMToBPSK (pm_pll -> pm_out)
void Demod::run_pll(const float2 *in, float2 *out, long n, float bw, float max_offset, int cur, int nxt)
{
    DemodDevState *S = st.p;
    const int L = choose_L(n);
    const int nseg = (int)((n + L - 1) / L);
    const int nblk = (nseg + SEG_THREADS - 1) / SEG_THREADS;
    PllParams P;
    { // pll_carrier_tracking.cpp:17-21
        float damping = sqrtf(2.0f) / 2.0f;
        float denom = (float)(1.0 + 2.0 * damping * bw + bw * bw);
        P.alpha = (4 * damping * bw) / denom;
        P.beta = (4 * bw * bw) / denom;
    }
    P.fmax = max_offset; // PLLCarrierTrackingBlock(input, bw, max_offset, -max_offset)
    P.fmin = -max_offset;
    const float mt = repair_merge ? 1.0f / MERGE_TIGHTER : 0.0f;
    run_loop_stage(*this, nblk, [&](int grid, const int *list, const int *count, int round) {
        k_pll<<<grid, SEG_THREADS, PLL_SMEM_BYTES, stream>>>(in, n, L, Wp, nseg, P, S->pll[cur], d_atan_tab.p, out, crec.p, list, count, cck.p, mt * tol_pphase,
                                                             mt * tol_pfreq, S->merge_hist);
        k_costas_fix<<<1, 1024, 0, stream>>>(crec.p, nseg, 1, tol_pphase, tol_pfreq, quad.p, S->pll[nxt], &S->pll_unconv, repair.p + 1, repair.p, round,
                                             &S->repairs);
    });
}

void Demod::stage_pll(long n, int cur, int nxt)
{
    run_pll(pm_agc.p, pm_pll.p, n, cfg.pm_pll_bw, cfg.pm_pll_max_offset, cur, nxt);
    run_rotator(pm_pll.p, B200_CF32, n, 0, 1, pm_dturn, pm_pos, pm_out.p);
    pm_pos += (unsigned long long)n;
}

// Costas loop (+ junction fix-up and repair rounds) over the FIR output in bufA, exact rotation / OQPSK delay / optional DC blocker
// into the clock recovery's input buffer (16-sample front pad: [8, 16) = the previous batch's last 8 inputs). Returns that buffer.
float2 *Demod::stage_costas(long n, int L, int nseg, int cur, int nxt, bool materialise)
{
    DemodDevState *S = st.p;
    mm_quad = nullptr;
    mm_rot = mm_oqpsk = 0;
    float2 *fir_out = bufA.p + 16, *cos_out = bufB.p + 16;
    const int nblk = (nseg + SEG_THREADS - 1) / SEG_THREADS;
    last_L = L;
    last_nseg = nseg;
    float2 *mmin;
    if (order && cfg.has_carrier) {
        // psk_demod carrier mode (module_psk_demod.cpp:109-112,121): carrier PLL on the RRC output, then CorrectIQBlock; the Costas loop
        // reads the result (written back over the RRC output)
        run_pll(fir_out, pm_pll.p, n, cfg.carrier_pll_bw, cfg.carrier_pll_max_offset, cur, nxt);
        run_dc(pm_pll.p, B200_CF32, 0, n, &S->dc_acc3[cur], &S->dc_acc3[nxt], fir_out);
    }
    if (order) {
        CostasParams P;
        P.order = order;
        { // costas_loop.cpp:5-12
            float damping = sqrtf(2.0f) / 2.0f;
            float denom = (float)(1.0 + 2.0 * damping * cfg.pll_bw + cfg.pll_bw * cfg.pll_bw);
            P.alpha = (4 * damping * cfg.pll_bw) / denom;
            P.beta = (4 * cfg.pll_bw * cfg.pll_bw) / denom;
        }
        P.fmin = -cfg.costas_max_offset;
        P.fmax = cfg.costas_max_offset;
        const auto costas = order == 2 ? k_costas<2> : (order == 4 ? k_costas<4> : k_costas<8>);
        const float mt = repair_merge ? 1.0f / MERGE_TIGHTER : 0.0f;
        run_loop_stage(*this, nblk, [&](int grid, const int *list, const int *count, int round) {
            costas<<<grid, SEG_THREADS, COSTAS_SMEM_BYTES, stream>>>(fir_out, n, L, Wc, Gc, nseg, P, S->costas[cur], cos_out, crec.p, list, count, cck.p,
                                                                     mt * tol_cphase, mt * tol_cfreq, S->merge_hist);
            k_costas_fix<<<1, 1024, 0, stream>>>(crec.p, nseg, order, tol_cphase, tol_cfreq, quad.p, S->costas[nxt], &S->costas_unconv, repair.p + 1, repair.p,
                                                 round, &S->repairs);
        });
        if (!materialise && !cfg.post_costas_dc) {
            // fused: the clock recovery rotates (and, for OQPSK, delays) its input rows itself
            k_mm_prep<<<1, 32, 0, stream>>>(bufB.p, n, L, order, quad.p, S->mm_hist[cur], S->mm_hist[nxt]);
            launches += 1;
            mm_quad = quad.p;
            mm_rot = order;
            mm_oqpsk = cfg.constellation == B200_OQPSK;
            return bufB.p;
        }
        mmin = bufA.p; // FIR output is dead now: reuse its buffer (in place compatible: same index mapping)
        k_rotate<<<2048, 256, 0, stream>>>(cos_out, n, L, order, cfg.constellation == B200_OQPSK, quad.p, S->mm_hist[cur], S->mm_hist[nxt], mmin);
        launches += 1;
        if (cfg.post_costas_dc) {
            // CorrectIQBlock on the loop's output (module_psk_demod.cpp:127-134); the clock recovery's 8-sample history are ITS outputs
            run_dc(mmin + 16, B200_CF32, 0, n, &S->dc_acc2[cur], &S->dc_acc2[nxt], pdc_out.p + 16);
            B200_CUDA(cudaMemcpyAsync(pdc_out.p + 16 - MM_HIST, S->pdc_hist[cur], MM_HIST * sizeof(float2), cudaMemcpyDeviceToDevice, stream));
            B200_CUDA(cudaMemcpyAsync(S->pdc_hist[nxt], pdc_out.p + 16 + n - MM_HIST, MM_HIST * sizeof(float2), cudaMemcpyDeviceToDevice, stream));
            mmin = pdc_out.p;
        }
    } else if (!materialise) {
        k_mm_prep<<<1, 32, 0, stream>>>(bufA.p, n, L, 0, quad.p, S->mm_hist[cur], S->mm_hist[nxt]);
        launches += 1;
        return bufA.p; // the clock recovery reads the FIR output in place
    } else {
        mmin = bufB.p;
        k_rotate<<<2048, 256, 0, stream>>>(fir_out, n, L, 0, 0, quad.p, S->mm_hist[cur], S->mm_hist[nxt], mmin);
        launches += 1;
    }
    return mmin;
}

// M&M clock recovery over mmin (+ stitching, repair rounds, compaction and the int8 quantiser). `strict`: test hook, see k_mm.
// all_symbols: every symbol lands in sym_out (b200_demod_pull_symbols reads them); otherwise only the tail the SNR estimate reads.
void Demod::stage_mm(float2 *mmin, long n, int L, int nseg, int cur, int nxt, int8_t *sdst, bool strict, bool all_symbols)
{
    DemodDevState *S = st.p;
    const int nblk = (nseg + SEG_THREADS - 1) / SEG_THREADS;
    const auto mm = mm_kernel(strict, cfg.clock_recovery == 1, mm_rot || mm_oqpsk, fsk);
    MMParams MP;
    MP.omega_mid = sps;
    MP.omega_limit = cfg.clock_omega_limit * sps;
    MP.omega_gain = cfg.clock_gain_omega;
    MP.mu_gain = cfg.clock_gain_mu;
    const int cap = slot_cap_for(L);
    const float mt = repair_merge ? 1.0f / MERGE_TIGHTER : 0.0f;
    B200_REQUIRE((size_t)nseg * cap <= slots.n, B200_ENOMEM, "internal: symbol slot storage too small");
    run_loop_stage(*this, nblk, [&](int grid, const int *list, const int *count, int round) {
        mm<<<grid, SEG_THREADS, MM_SMEM_BYTES, stream>>>(mmin, n, L, Wm, Gm, nseg, MP, &S->mm[cur], &S->mm[nxt], d_bank.p, slots.p, cap, mrec.p, list, count,
                                                        mm_quad, mm_rot, mm_oqpsk, mck.p, mt * tol_mm, mt * tol_momega, S->merge_hist);
        k_mm_scan<<<1, 1024, 0, stream>>>(mrec.p, nseg, tol_mm, offs.p, &S->mm_unconv, cap, &S->flags, repair.p + 1, repair.p, round, &S->repairs);
    });
    k_mm_compact<<<std::min(nseg, 132 * 8), 256, 0, stream>>>(slots.p, cap, mrec.p, offs.p, nseg, fsk ? 3 : (pm ? 2 : (bps == 1)), all_symbols ? 1 : 0,
                                                              sym_out.p, sdst);
    // M2M4SNREstimator(alpha = 0.001); fsk_demod estimates over its float symbols taken as complex pairs (module_fsk_demod.cpp:127)
    k_snr_m2m4<<<1, 1024, 0, stream>>>(sym_out.p, offs.p + nseg, fsk ? 1 : 0, 0.001f, S->snr_y[cur], S->snr_y[nxt]);
    launches += 2;
}

// SmartResamplerBlock (module_demod_base.cpp:203-204; behind PMToBPSK for pm_demod with resample_after_pll): power-of-two decimator
// stages, then the rational resampler. Updates (d_raw, n, front_fmt) to the stage's output; rs_swap: the reader's iq_swap still to apply.
void Demod::front_resample(const void *&d_raw, long &n, int &front_fmt, int &rs_swap, long n_in, int cur, int nxt)
{
    DemodDevState *S = st.p;
    for (auto &stg : decim) {
        // outputs of this batch: all j >= 0 with inc + j * D < n (the for loop of decimating_fir.cpp:66-76)
        long J = 0;
        if (n > stg.inc)
            J = (n - stg.inc + stg.D - 1) / stg.D;
        B200_REQUIRE(J >= 64, B200_ESTATE, "batch of %ld samples decimates to %ld: push at least %d samples", n_in, J, 64 * decim_total + 4096);
        const unsigned grid = (unsigned)((std::max<long>(J, stg.nt) + 255) / 256);
        with_fmt(front_fmt, [&](auto F) {
            k_decim_fir<F><<<grid, 256, 0, stream>>>(d_raw, n, rs_swap, stg.tail[cur].p, stg.tail[nxt].p, stg.d_taps.p, stg.nt, stg.D, stg.inc, J, stg.out.p);
        });
        launches++;
        stg.inc = stg.inc + J * stg.D - n;
        d_raw = stg.out.p;
        n = J;
        front_fmt = B200_CF32;
        rs_swap = 0;
    }
    if (resamp && !((cfg.dc_block || !decim.empty()) && rs_I == 1 && rs_D == 1 && rs_nt == 1)) {
        // outputs of this batch: all j >= 0 with rs_inc + (rs_ctr + j*D) / I < n  (the while loop of rational_resampler.cpp:48-57)
        const long I = rs_I, D = rs_D;
        long J = 0;
        if (n > rs_inc)
            J = ((n - rs_inc) * I - rs_ctr + D - 1) / D;
        B200_REQUIRE(J >= 64 && J <= max_work, B200_ESTATE, "batch of %ld samples resamples to %ld: outside [64, %ld]", n, J, max_work);
        const unsigned grid = (unsigned)((J + RS_THREADS - 1) / RS_THREADS);
        with_fmt(front_fmt, [&](auto F) {
            k_resample<F><<<grid, RS_THREADS, 0, stream>>>(d_raw, n, rs_swap, S->rs_tail[cur], S->rs_tail[nxt], d_rs_bank.p, rs_I, rs_D, rs_nt, rs_inc, rs_ctr, J,
                                                          rs_out.p);
        });
        launches++;
        const long c_end = rs_ctr + J * D;
        rs_inc = rs_inc + c_end / I - n;
        rs_ctr = c_end % I;
        d_raw = rs_out.p;
        n = J;
        front_fmt = B200_CF32;
    }
}

// fsk_demod behind the complex AGC (pm_agc): QuadratureDemodBlock -> CorrectIQBlock<float> -> AGCBlock<float> (both scanned over tiles from
// the carried accumulator / gain) -> FIRBlock<float> with its carried history -> the clock recovery's input (y, 0) in bufA + 16
void Demod::stage_fsk(long n, const FirTaps &taps, int cur, int nxt)
{
    DemodDevState *S = st.p;
    const int nt = (int)((n + FIR_TILE - 1) / FIR_TILE);
    const float alpha = 0.0001f, beta = 1.0f - alpha; // CorrectIQBlock<float> (correct_iq.h:23, correct_iq.cpp:9)
    k_quad<<<nt, FIR_THREADS, 0, stream>>>(pm_agc.p, n, &S->qphase[cur], &S->qphase[nxt], alpha, beta, quad_out.p, tile_map.p);
    k_tile_scan<<<1, 1024, 0, stream>>>(tile_map.p, nt, &S->fdc_acc[cur], nullptr, 0, seeds.p, nullptr);
    k_fsk_dc<<<nt, FIR_THREADS, 0, stream>>>(quad_out.p, n, alpha, beta, seeds.p, dc2_out.p, &S->fdc_acc[nxt], tile_map3.p);
    k_tile_scan<<<1, 1024, 0, stream>>>(tile_map3.p, nt, &S->fgain[cur], nullptr, 0, seeds.p, nullptr);
    k_fsk_agc<<<nt, FIR_THREADS, 0, stream>>>(dc2_out.p, n, seeds.p, agc2_out.p + 32, &S->fgain[nxt]);
    B200_CUDA(cudaMemcpyAsync(agc2_out.p, S->fir_tail[cur], 32 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    k_fir_real<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(agc2_out.p + 32, n, taps, bufA.p + 16);
    B200_CUDA(cudaMemcpyAsync(S->fir_tail[nxt], agc2_out.p + n, 32 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    launches += 6;
}

long Demod::process(const void *d_raw, long n, int8_t *soft_dst)
{
    B200_REQUIRE(n >= 64, B200_ESTATE, "a batch needs at least 64 samples (got %ld)", n);
    B200_REQUIRE(n <= max_batch, B200_ESTATE, "batch of %ld samples exceeds max_batch %ld", n, max_batch);
    DeviceGuard g(cfg.device);
    const int cur = parity, nxt = parity ^ 1;
    DemodDevState *S = st.p;
    const long n_in = n;
    last_in = n;
    int front_fmt = cfg.format;
    B200_CUDA(cudaMemsetAsync(&S->flags, 0, sizeof(int), stream)); // per-batch conditions (AGC clamp seen, slot overflow)
    B200_CUDA(cudaEventRecord(ev[0], stream));
    int rs_swap = cfg.iq_swap;
    if (cfg.dc_block) {
        // CorrectIQBlock sits right behind the reader (module_demod_base.cpp:113-120): (iq_swap ->) dc block -> (resampler ->) AGC
        run_dc(d_raw, cfg.format, cfg.iq_swap, n, &S->dc_acc[cur], &S->dc_acc[nxt], dc_out.p);
        d_raw = dc_out.p;
        front_fmt = B200_CF32;
        rs_swap = 0; // already applied
    }
    if (cfg.freq_shift != 0) {
        // FreqShiftBlock behind the DC blocker, in front of the resampler (module_demod_base.cpp:122-123,203)
        run_rotator(d_raw, front_fmt, n, rs_swap, 0, fs_dturn, fs_pos, fs_out.p);
        fs_pos += (unsigned long long)n;
        d_raw = fs_out.p;
        front_fmt = B200_CF32;
        rs_swap = 0;
    }
    if (!pm_after) // initb(!d_resample_after_pll) (module_pm_demod.cpp:63)
        front_resample(d_raw, n, front_fmt, rs_swap, n_in, cur, nxt);
    else if (rs_swap) { // the reader's swap, which the front-end kernels would have applied: a plain converting copy
        run_rotator(d_raw, front_fmt, n, 1, 0, 0ull, 0ull, pm_out.p);
        d_raw = pm_out.p;
        front_fmt = B200_CF32;
        rs_swap = 0;
    }
    last_front = n;
    FirTaps taps;
    memset(&taps, 0, sizeof(taps));
    for (int i = 0; i < FIR_NT; i++)
        taps.h[i] = rrc[i];
    const bool dump = cfg.keep_stages != 0;
    if (fsk) {
        // the complex AGC runs through the front kernel with its output dumped (the FIR it also computes is not used)
        const AgcUnit u{cfg.agc_rate, 65536.0f, &S->gain[cur], &S->gain[nxt], S->agc_tail[cur], S->agc_tail[nxt], bufA.p + 16, pm_agc.p};
        launch_front_fmt(*this, front_fmt, d_raw, n, taps, u);
        stage_fsk(n, taps, cur, nxt);
    } else if (!pm) {
        const AgcUnit u{cfg.agc_rate, 65536.0f, &S->gain[cur], &S->gain[nxt], S->agc_tail[cur], S->agc_tail[nxt], bufA.p + 16, dump ? agc_dump.p : nullptr};
        launch_front_fmt(*this, front_fmt, d_raw, n, taps, u);
    } else {
        // pm_demod (module_pm_demod.cpp:61-88): AGC -> carrier PLL -> PMToBPSK -> [resampler -> AGC2] -> RRC. The first AGC runs through
        // the same kernel with its output dumped (the FIR it also computes is not used)
        const AgcUnit u1{cfg.agc_rate, 65536.0f, &S->gain[cur], &S->gain[nxt], S->agc1_tail[cur], S->agc1_tail[nxt], bufA.p + 16, pm_agc.p};
        launch_front_fmt(*this, front_fmt, d_raw, n, taps, u1);
        stage_pll(n, cur, nxt);
        last_pm = n;
        d_raw = pm_out.p;
        front_fmt = B200_CF32;
        if (pm_after) {
            front_resample(d_raw, n, front_fmt, rs_swap, n_in, cur, nxt);
            last_front = n;
            // agc2 = AGCBlock(resampler->output_stream, 0.001, 1.0, 1.0, 1000.0) (module_pm_demod.cpp:73-74)
            const AgcUnit u2{0.001f, 1000.0f, &S->gain2[cur], &S->gain2[nxt], S->agc2_tail[cur], S->agc2_tail[nxt], bufA.p + 16, dump ? agc_dump.p : nullptr};
            launch_front_fmt(*this, front_fmt, d_raw, n, taps, u2);
        } else {
            // the RRC reads PMToBPSK's output directly: rate 0 makes every AGC step the identity map and the gain stay 1
            const AgcUnit u2{0.0f, 65536.0f, &S->gain2[cur], &S->gain2[nxt], S->agc2_tail[cur], S->agc2_tail[nxt], bufA.p + 16, nullptr};
            launch_front_fmt(*this, front_fmt, d_raw, n, taps, u2);
        }
    }
    B200_CUDA(cudaEventRecord(ev[1], stream));
    float2 *fir_out = bufA.p + 16, *cos_out = bufB.p + 16;
    if (dump || keep_front)
        B200_CUDA(cudaMemcpyAsync(fir_dump.p, fir_out, n * sizeof(float2), cudaMemcpyDeviceToDevice, stream));

    const int L = choose_L(n);
    const int nseg = (int)((n + L - 1) / L);
    float2 *mmin = stage_costas(n, L, nseg, cur, nxt, cfg.keep_stages != 0);
    B200_CUDA(cudaEventRecord(ev[2], stream));
    // a caller-supplied soft destination (the fused chain) consumes the soft stream only: its demodulator's symbols are never pulled
    stage_mm(mmin, n, L, nseg, cur, nxt, soft_dst ? soft_dst : soft.p, false, soft_dst == nullptr);
    B200_CUDA(cudaEventRecord(ev[3], stream));
    B200_CUDA(cudaMemcpyAsync(h_total.p, offs.p + nseg, sizeof(long), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(h_state.p, st.p, sizeof(DemodDevState), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&t_agcfir, ev[0], ev[1]);
    cudaEventElapsedTime(&t_costas, ev[1], ev[2]);
    cudaEventElapsedTime(&t_mm, ev[2], ev[3]);
    parity = nxt;
    last_n = n;
    last_syms = *h_total.p;
    total_in += n_in;
    total_syms += last_syms;
    {
        // M2M4SNREstimator::snr (snr_estimator.cpp:41-47), float arithmetic as there
        const float y1 = h_state.p->snr_y[nxt][0], y2 = h_state.p->snr_y[nxt][1];
        const float y1_2 = y1 * y1;
        const float sig = (float)sqrt(2 * y1_2 - y2), noise = (float)(y1 - sqrt(2 * y1_2 - y2));
        snr_now = std::max<float>(0, (float)(10.0 * log10(sig / noise)));
        if (!(snr_now == snr_now))
            snr_now = 0.f;
        if (snr_now > snr_peak)
            snr_peak = snr_now;
    }
    if (h_state.p->flags & 1)
        agc_clamped_batches++; // the clamp pass produced this batch's front stage (silent input): information, not an error
    if (h_state.p->flags & 2)
        throw ApiError(B200_EUNSUPPORTED, "M&M produced more symbols per segment than the omega limit allows (slot overflow)");
    return last_syms;
}

// Test hook behind b200_demod_debug_run_stage: ONE stage of a freshly reset demodulator on a caller-supplied cf32 stage input.
long Demod::debug_run_stage(int stage, const float *h_in, long n, int mode, float *h_out, long cap)
{
    B200_REQUIRE(n >= 64 && n <= max_work, B200_ESTATE, "stage input of %ld samples outside [64, %ld]", n, max_work);
    if (fsk)
        return debug_run_stage_fsk(stage, h_in, n, mode, h_out, cap);
    B200_REQUIRE(stage == B200_STAGE_FIR || stage == B200_STAGE_COSTAS || stage == B200_STAGE_MM || stage == B200_STAGE_PLL || stage == B200_STAGE_PM, B200_EINVAL,
                 "stage %d cannot be run alone", stage);
    DeviceGuard g(cfg.device);
    reset();
    const bool strict = mode & B200_DEBUG_STRICT, seq = mode & B200_DEBUG_SEQUENTIAL;
    const int L = seq ? (int)((n + 15) / 16 * 16) : choose_L(n);
    const int nseg = (int)((n + L - 1) / L);
    DemodDevState *S = st.p;
    long count = n;
    const float2 *src = nullptr;
    if (stage == B200_STAGE_FIR) {
        FirTaps taps;
        memset(&taps, 0, sizeof(taps));
        for (int i = 0; i < FIR_NT; i++)
            taps.h[i] = rrc[i];
        B200_CUDA(cudaMemcpyAsync(bufB.p + 16, h_in, n * sizeof(float2), cudaMemcpyHostToDevice, stream));
        if (strict)
            k_fir_only<true><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(bufB.p + 16, n, taps, bufA.p + 16);
        else {
            // the production kernel with the AGC switched off: rate 0 makes every step map the identity and the gain stay 1, so
            // k_agc_fir_w's output is the FFMA FIR of its input (the ranges take the scanned-seed pass: nothing proves a seed at rate 0)
            const AgcUnit u{0.0f, 65536.0f, &S->gain[0], &S->gain[1], S->agc_tail[0], S->agc_tail[1], bufA.p + 16, nullptr};
            launch_front_fmt(*this, B200_CF32, bufB.p + 16, n, taps, u);
        }
        src = bufA.p + 16;
    } else if (stage == B200_STAGE_PLL || stage == B200_STAGE_PM) {
        // pm_demod's carrier PLL on a caller-supplied AGC output (SEQUENTIAL: one segment = the reference's loop, bit for bit), and
        // PMToBPSK behind it
        B200_REQUIRE(pm, B200_EINVAL, "this configuration is not a pm_demod");
        B200_CUDA(cudaMemcpyAsync(pm_agc.p, h_in, n * sizeof(float2), cudaMemcpyHostToDevice, stream));
        const int keep = seg_cap_threads;
        if (seq)
            seg_cap_threads = 1; // choose_L: one segment as long as allowed; longer inputs still split (use <= 16384 samples for the bitwise check)
        stage_pll(n, 0, 1);
        seg_cap_threads = keep;
        src = stage == B200_STAGE_PLL ? pm_pll.p : pm_out.p;
    } else if (stage == B200_STAGE_COSTAS) {
        B200_REQUIRE(order != 0, B200_EINVAL, "this configuration has no Costas loop");
        B200_CUDA(cudaMemcpyAsync(bufA.p + 16, h_in, n * sizeof(float2), cudaMemcpyHostToDevice, stream));
        src = stage_costas(n, L, nseg, 0, 1, true) + 16;
    } else {
        float2 *mmin = order ? bufA.p : bufB.p;
        mm_quad = nullptr; // the stage input is the clock recovery's input as it is: no rotation, no delay
        mm_rot = mm_oqpsk = 0;
        B200_CUDA(cudaMemsetAsync(mmin, 0, 16 * sizeof(float2), stream)); // history of a new stream
        B200_CUDA(cudaMemcpyAsync(mmin + 16, h_in, n * sizeof(float2), cudaMemcpyHostToDevice, stream));
        last_L = L;
        last_nseg = nseg;
        stage_mm(mmin, n, L, nseg, 0, 1, soft.p, strict, true);
        B200_CUDA(cudaMemcpyAsync(h_total.p, offs.p + nseg, sizeof(long), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        count = *h_total.p;
        src = sym_out.p;
    }
    B200_REQUIRE(count <= cap, B200_ESTATE, "output buffer too small: need %ld complex values", count);
    B200_CUDA(cudaMemcpyAsync(h_out, src, count * sizeof(float2), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(h_state.p, S, sizeof(DemodDevState), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    dbg_costas_unconv = (stage == B200_STAGE_PLL || stage == B200_STAGE_PM) ? h_state.p->pll_unconv : h_state.p->costas_unconv;
    dbg_mm_unconv = h_state.p->mm_unconv;
    dbg_repairs = h_state.p->repairs;
    last_syms = stage == B200_STAGE_MM ? count : 0;
    reset();
    return count;
}

// debug_run_stage of an fsk_demod: every stage input and output is one float per sample (QUAD: complex input)
long Demod::debug_run_stage_fsk(int stage, const float *h_in, long n, int mode, float *h_out, long cap)
{
    B200_REQUIRE(stage == B200_STAGE_QUAD || stage == B200_STAGE_DC2 || stage == B200_STAGE_AGC2 || stage == B200_STAGE_FIR || stage == B200_STAGE_MM,
                 B200_EINVAL, "stage %d cannot be run alone in fsk_demod", stage);
    const bool strict = mode & B200_DEBUG_STRICT, seq = mode & B200_DEBUG_SEQUENTIAL;
    B200_REQUIRE(seq || (stage != B200_STAGE_DC2 && stage != B200_STAGE_AGC2), B200_EINVAL,
                 "fsk_demod runs its DC blocker and AGC alone only as SEQUENTIAL (the scanned ones run inside a push with keep_stages)");
    DeviceGuard g(cfg.device);
    reset();
    DemodDevState *S = st.p;
    const float alpha = 0.0001f, beta = 1.0f - alpha;
    float *in = agc2_out.p + 32; // real stage inputs, behind a zero history
    const float *src = nullptr;
    long count = n;
    if (stage == B200_STAGE_QUAD) {
        B200_CUDA(cudaMemcpyAsync(pm_agc.p, h_in, n * sizeof(float2), cudaMemcpyHostToDevice, stream));
        k_quad<<<(unsigned)((n + FIR_TILE - 1) / FIR_TILE), FIR_THREADS, 0, stream>>>(pm_agc.p, n, &S->qphase[0], &S->qphase[1], alpha, beta, quad_out.p,
                                                                                     tile_map.p);
        src = quad_out.p;
    } else if (stage == B200_STAGE_MM) {
        // the clock recovery's input (x, 0) with a zero history, as k_fir_real writes it
        const int L = seq ? (int)((n + 15) / 16 * 16) : choose_L(n);
        const int nseg = (int)((n + L - 1) / L);
        mm_quad = nullptr;
        mm_rot = mm_oqpsk = 0;
        B200_CUDA(cudaMemsetAsync(bufA.p, 0, (n + 16) * sizeof(float2), stream));
        B200_CUDA(cudaMemcpy2DAsync(bufA.p + 16, sizeof(float2), h_in, sizeof(float), sizeof(float), n, cudaMemcpyHostToDevice, stream));
        last_L = L;
        last_nseg = nseg;
        stage_mm(bufA.p, n, L, nseg, 0, 1, soft.p, strict, true);
        B200_CUDA(cudaMemcpyAsync(h_total.p, offs.p + nseg, sizeof(long), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        count = *h_total.p;
        src = reinterpret_cast<const float *>(sym_out.p);
    } else {
        B200_CUDA(cudaMemsetAsync(agc2_out.p, 0, 32 * sizeof(float), stream));
        B200_CUDA(cudaMemcpyAsync(in, h_in, n * sizeof(float), cudaMemcpyHostToDevice, stream));
        if (stage == B200_STAGE_FIR) {
            FirTaps taps;
            memset(&taps, 0, sizeof(taps));
            for (int i = 0; i < FIR_NT; i++)
                taps.h[i] = rrc[i];
            k_fir_real<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(in, n, taps, bufA.p + 16);
            B200_CUDA(cudaMemcpy2DAsync(quad_out.p, sizeof(float), bufA.p + 16, sizeof(float2), sizeof(float), n, cudaMemcpyDeviceToDevice, stream));
            src = quad_out.p;
        } else {
            k_fsk_serial<<<1, 1, 0, stream>>>(stage == B200_STAGE_DC2 ? 0 : 1, in, n, alpha, beta, dc2_out.p);
            src = dc2_out.p;
        }
    }
    B200_REQUIRE(count <= cap, B200_ESTATE, "output buffer too small: need %ld values", count);
    B200_CUDA(cudaMemcpyAsync(h_out, src, count * sizeof(float), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(h_state.p, S, sizeof(DemodDevState), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    dbg_costas_unconv = 0;
    dbg_mm_unconv = h_state.p->mm_unconv;
    dbg_repairs = h_state.p->repairs;
    last_syms = stage == B200_STAGE_MM ? count : 0;
    reset();
    return count;
}

void Demod::prefetch_host(const void *h_raw, long n)
{
    B200_REQUIRE(n <= max_batch && n >= 64, B200_ESTATE, "prefetch of %ld samples outside [64, max_batch %ld]", n, max_batch);
    DeviceGuard g(cfg.device);
    const int bytes = fmt_bytes(cfg.format);
    if (!raw2.p)
        raw2.alloc((size_t)max_batch * bytes + 64);
    Prefetch *slot = !pf[0].valid ? &pf[0] : (!pf[1].valid ? &pf[1] : nullptr);
    B200_REQUIRE(slot != nullptr, B200_ESTATE, "two prefetched batches are already pending: push one first");
    // the staging buffer no pending prefetch occupies (pushes may come in any order, so a blind alternation could overwrite one)
    const Prefetch *other = slot == &pf[0] ? &pf[1] : &pf[0];
    slot->buf = (other->valid && other->buf == 0) ? 1 : 0;
    B200_CUDA(cudaMemcpyAsync(slot->buf ? raw2.p : raw.p, h_raw, (size_t)n * bytes, cudaMemcpyHostToDevice, copy_stream));
    B200_CUDA(cudaEventRecord(slot->done, copy_stream));
    slot->ptr = h_raw;
    slot->n = n;
    slot->valid = true;
    slot->seq = pf_seq++;
}

long Demod::push_host(const void *h_raw, long n, int8_t *soft_dst)
{
    B200_REQUIRE(n <= max_batch, B200_ESTATE, "batch of %ld samples exceeds max_batch %ld", n, max_batch);
    DeviceGuard g(cfg.device);
    // oldest matching prefetch, if any
    Prefetch *hit = nullptr;
    for (auto &p : pf)
        if (p.valid && p.ptr == h_raw && p.n == n && (!hit || p.seq < hit->seq))
            hit = &p;
    if (hit) {
        B200_CUDA(cudaStreamWaitEvent(stream, hit->done, 0));
        hit->valid = false;
        return process(hit->buf ? raw2.p : raw.p, n, soft_dst);
    }
    const int bytes = fmt_bytes(cfg.format);
    // no pending prefetch may target the buffer we copy into
    unsigned char *dst = (pf[0].valid && pf[0].buf == 0) || (pf[1].valid && pf[1].buf == 0) ? nullptr : raw.p;
    if (!dst) {
        if (!raw2.p)
            raw2.alloc((size_t)max_batch * bytes + 64);
        B200_REQUIRE(!((pf[0].valid && pf[0].buf == 1) || (pf[1].valid && pf[1].buf == 1)), B200_ESTATE, "both staging buffers hold prefetched batches");
        dst = raw2.p;
    }
    B200_CUDA(cudaMemcpyAsync(dst, h_raw, (size_t)n * bytes, cudaMemcpyHostToDevice, stream));
    return process(dst, n, soft_dst);
}

void Demod::stats(b200_demod_stats *o)
{
    memset(o, 0, sizeof(*o));
    o->samples_in = total_in;
    o->symbols_out = total_syms;
    o->agc_gain = h_state.p->gain[parity];
    o->costas_phase = h_state.p->costas[parity][0];
    o->costas_freq = h_state.p->costas[parity][1];
    o->mm_mu = h_state.p->mm[parity].mu;
    o->mm_omega = h_state.p->mm[parity].omega;
    o->costas_unconverged = h_state.p->costas_unconv;
    o->mm_unconverged = h_state.p->mm_unconv;
    o->agc_clamped = (int)std::min<long>(agc_clamped_batches, 0x7fffffff); // batches in which the gain hit max_gain so far
    o->repairs = h_state.p->repairs;
    for (int i = 0; i < MERGE_BUCKETS; i++)
        o->repair_merge_hist[i] = h_state.p->merge_hist[i];
    o->kernel_launches = launches;
    o->agc_exact_passes = h_state.p->agc_exact;
    o->last_front_samples = last_front;
    o->snr = snr_now;
    o->peak_snr = snr_peak;
    o->pll_freq = (pm || cfg.has_carrier) ? h_state.p->pll[parity][1] : 0.f;
    o->pll_unconverged = (pm || cfg.has_carrier) ? h_state.p->pll_unconv : 0;
    o->last_range_tiles = last_R;
}

} // namespace b200

using namespace b200;
struct b200_demod
{
    Demod *d;
};

extern "C" {
const char *b200_last_error(void) { return b200::last_error_cstr(); }
int b200_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess)
        return 0;
    return n;
}

b200_demod *b200_demod_create(const b200_demod_cfg *cfg)
{
    b200_demod *h = nullptr;
    int rc = guarded([&] {
        B200_REQUIRE(cfg != nullptr, B200_EINVAL, "cfg is NULL");
        h = new b200_demod{new Demod(*cfg)};
    });
    (void)rc;
    return h;
}
void b200_demod_destroy(b200_demod *h)
{
    if (!h)
        return;
    delete h->d;
    delete h;
}
int b200_demod_push_iq(b200_demod *h, const void *host_iq, long n)
{
    return guarded([&] {
        B200_REQUIRE(h && host_iq, B200_EINVAL, "NULL argument");
        h->d->push_host(host_iq, n, nullptr);
    });
}
int b200_demod_push_iq_device(b200_demod *h, const void *dev_iq, long n)
{
    return guarded([&] {
        B200_REQUIRE(h && dev_iq, B200_EINVAL, "NULL argument");
        h->d->process(dev_iq, n, nullptr);
    });
}
int b200_demod_pull_soft(b200_demod *h, int8_t *out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        Demod &d = *h->d;
        long nb = d.last_syms * d.bps;
        B200_REQUIRE(nb <= cap, B200_ESTATE, "output buffer too small: need %ld bytes", nb);
        DeviceGuard g(d.cfg.device);
        B200_CUDA(cudaMemcpyAsync(out, d.soft.p, nb, cudaMemcpyDeviceToHost, d.stream));
        B200_CUDA(cudaStreamSynchronize(d.stream));
        *n_out = nb;
    });
}
int b200_demod_pull_symbols(b200_demod *h, float *out, long cap_symbols, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        Demod &d = *h->d;
        B200_REQUIRE(d.last_syms <= cap_symbols, B200_ESTATE, "output buffer too small: need %ld symbols", d.last_syms);
        DeviceGuard g(d.cfg.device);
        B200_CUDA(cudaMemcpyAsync(out, d.sym_out.p, d.last_syms * (d.fsk ? sizeof(float) : sizeof(float2)), cudaMemcpyDeviceToHost, d.stream));
        B200_CUDA(cudaStreamSynchronize(d.stream));
        *n_out = d.last_syms;
    });
}
double b200_demod_final_samplerate(double samplerate, double symbolrate, int constellation, float min_sps, float max_sps, double custom_samplerate)
{
    // module_demod_base.cpp:59-80 with its types: long d_samplerate, int d_symbolrate, float MIN_SPS / MAX_SPS / final_samplerate
    const long d_samplerate = (long)samplerate;
    const int d_symbolrate = (int)symbolrate;
    const SpsWindow win = sps_window(constellation, min_sps, max_sps);
    const float MIN_SPS = win.lo, MAX_SPS = win.hi;
    if (d_symbolrate <= 0 || d_samplerate <= 0)
        return samplerate;
    const float input_sps = (float)d_samplerate / (float)d_symbolrate;
    const bool resample = input_sps > MAX_SPS || input_sps < MIN_SPS;
    const int range = (int)pow(10, (std::to_string(int(d_symbolrate)).size() - 1));
    float final_samplerate = (float)d_samplerate;
    if (custom_samplerate > 0)
        final_samplerate = (float)(long)custom_samplerate;
    else if (MAX_SPS == MIN_SPS)
        final_samplerate = d_symbolrate * MAX_SPS;
    else if (input_sps > MAX_SPS)
        final_samplerate = resample ? (round(d_symbolrate / range) * range) * MAX_SPS : d_samplerate;
    else if (input_sps < MIN_SPS)
        final_samplerate = resample ? d_symbolrate * MIN_SPS : d_samplerate;
    return (double)final_samplerate;
}
int b200_demod_resample_decision(double samplerate, double symbolrate, int constellation, float min_sps, float max_sps)
{
    const long d_samplerate = (long)samplerate;
    const int d_symbolrate = (int)symbolrate;
    const SpsWindow win = sps_window(constellation, min_sps, max_sps);
    if (d_symbolrate <= 0 || d_samplerate <= 0)
        return 0;
    const float input_sps = (float)d_samplerate / (float)d_symbolrate;
    return (input_sps > win.hi || input_sps < win.lo) ? 1 : 0;
}
int b200_demod_resampler_bank(double samplerate, double final_samplerate, float *out, long cap, int *ntaps, int *interp, int *decim)
{
    return guarded([&] {
        B200_REQUIRE(out && ntaps && interp && decim, B200_EINVAL, "NULL argument");
        // the constructor's reduction: the rational part behind the power-of-two decimator -> RationalResamplerBlock::set_ratio
        const unsigned interpolation = (unsigned)(float)final_samplerate, decimation = (unsigned)(long)samplerate;
        B200_REQUIRE(interpolation > 0 && decimation > 0, B200_EINVAL, "rates must be positive");
        const SmartRatio r = smart_resampler_ratio(interpolation, decimation);
        std::vector<float> bank;
        const int nt = design_resampler_bank(r.I, r.D, bank);
        B200_REQUIRE((long)bank.size() <= cap, B200_ESTATE, "output buffer too small: need %zu floats", bank.size());
        memcpy(out, bank.data(), bank.size() * sizeof(float));
        *ntaps = nt;
        *interp = (int)r.I;
        *decim = (int)r.D;
    });
}
int b200_demod_debug_stage(b200_demod *h, int stage, float *out, long cap_samples)
{
    return guarded([&] {
        B200_REQUIRE(h && out, B200_EINVAL, "NULL argument");
        Demod &d = *h->d;
        B200_REQUIRE(d.cfg.keep_stages || (d.keep_front && stage == B200_STAGE_FIR), B200_ESTATE,
                     "create the demodulator with keep_stages=1 to read stage outputs (or set keep_front for the RRC output)");
        // pm_demod: the first AGC, the carrier PLL and PMToBPSK run on last_pm samples (the input rate with resample_after_pll)
        const bool at_pll = d.pm && (stage == B200_STAGE_AGC || stage == B200_STAGE_PLL || stage == B200_STAGE_PM);
        const long count = stage == B200_STAGE_DC ? d.last_in : (at_pll ? d.last_pm : d.last_n);
        B200_REQUIRE(count <= cap_samples, B200_ESTATE, "output buffer too small");
        if (d.fsk && stage != B200_STAGE_AGC && stage != B200_STAGE_RESAMP && stage != B200_STAGE_DC) {
            // fsk_demod's real stages: one float per sample (the FIR output is the .x of the clock recovery's input)
            DeviceGuard g(d.cfg.device);
            if (stage == B200_STAGE_FIR)
                B200_CUDA(cudaMemcpy2DAsync(out, sizeof(float), d.fir_dump.p, sizeof(float2), sizeof(float), count, cudaMemcpyDeviceToHost, d.stream));
            else {
                const float *fsrc = stage == B200_STAGE_QUAD ? d.quad_out.p : (stage == B200_STAGE_DC2 ? d.dc2_out.p : (stage == B200_STAGE_AGC2 ? d.agc2_out.p + 32 : nullptr));
                B200_REQUIRE(fsrc, B200_EINVAL, "unknown stage %d of fsk_demod", stage);
                B200_CUDA(cudaMemcpyAsync(out, fsrc, count * sizeof(float), cudaMemcpyDeviceToHost, d.stream));
            }
            B200_CUDA(cudaStreamSynchronize(d.stream));
            return;
        }
        const float2 *src = nullptr;
        if (stage == B200_STAGE_AGC)
            src = (d.pm || d.fsk) ? d.pm_agc.p : d.agc_dump.p;
        else if (stage == B200_STAGE_FIR)
            src = d.fir_dump.p;
        else if (stage == B200_STAGE_PLL && (d.pm || d.cfg.has_carrier))
            src = d.pm_pll.p; // carrier PLL output (as many samples as entered the PLL)
        else if (stage == B200_STAGE_PM && d.pm)
            src = d.pm_out.p; // PMToBPSK output
        else if (stage == B200_STAGE_COSTAS)
            src = (d.cfg.post_costas_dc ? d.pdc_out.p : (d.order ? d.bufA.p : d.bufB.p)) + 16; // M&M input = Costas output after rotation fix-up (+ post-Costas DC blocker / OQPSK delay)
        else if (stage == B200_STAGE_RESAMP && (d.resamp || !d.decim.empty()))
            src = d.resamp ? d.rs_out.p : d.decim.back().out.p; // what entered the AGC: front-end decimator / resampler / iq_swap output
        else if (stage == B200_STAGE_DC && d.cfg.dc_block)
            src = d.dc_out.p; // DC blocker output (as many samples as were pushed)
        B200_REQUIRE(src, B200_EINVAL, "unknown stage %d", stage);
        DeviceGuard g(d.cfg.device);
        B200_CUDA(cudaMemcpyAsync(out, src, count * sizeof(float2), cudaMemcpyDeviceToHost, d.stream));
        B200_CUDA(cudaStreamSynchronize(d.stream));
    });
}
int b200_demod_debug_convert(b200_demod *h, const void *host_iq, long n, float *host_out)
{
    return guarded([&] {
        B200_REQUIRE(h && host_iq && host_out, B200_EINVAL, "NULL argument");
        Demod &d = *h->d;
        B200_REQUIRE(n > 0 && n <= d.max_batch, B200_ESTATE, "sample count outside (0, max_batch]");
        DeviceGuard g(d.cfg.device);
        B200_CUDA(cudaMemcpyAsync(d.raw.p, host_iq, (size_t)n * fmt_bytes(d.cfg.format), cudaMemcpyHostToDevice, d.stream));
        float2 *out = d.bufB.p + 16;
        const unsigned blocks = (unsigned)((n + 8 * 256 - 1) / (8 * 256));
        with_fmt(d.cfg.format, [&](auto F) { k_convert_only<F><<<blocks, 256, 0, d.stream>>>(d.raw.p, n, out); });
        B200_CUDA(cudaMemcpyAsync(host_out, out, n * sizeof(float2), cudaMemcpyDeviceToHost, d.stream));
        B200_CUDA(cudaStreamSynchronize(d.stream));
    });
}
int b200_demod_debug_run_stage(b200_demod *h, int stage, const float *host_in, long n, int mode, float *host_out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && host_in && host_out && n_out, B200_EINVAL, "NULL argument");
        *n_out = h->d->debug_run_stage(stage, host_in, n, mode, host_out, cap);
    });
}
int b200_demod_debug_junctions(b200_demod *h, double *costas_out, double *mm_out, long cap_segments, long *nseg_out, long *seg_len)
{
    return guarded([&] {
        B200_REQUIRE(h && nseg_out && seg_len, B200_EINVAL, "NULL argument");
        Demod &d = *h->d;
        const long ns = d.last_nseg;
        B200_REQUIRE(ns <= cap_segments, B200_ESTATE, "output buffers too small: %ld segments", ns);
        DeviceGuard g(d.cfg.device);
        std::vector<LoopRec> cr(ns);
        std::vector<MMRec> mr(ns);
        B200_CUDA(cudaMemcpyAsync(cr.data(), d.crec.p, ns * sizeof(LoopRec), cudaMemcpyDeviceToHost, d.stream));
        B200_CUDA(cudaMemcpyAsync(mr.data(), d.mrec.p, ns * sizeof(MMRec), cudaMemcpyDeviceToHost, d.stream));
        B200_CUDA(cudaStreamSynchronize(d.stream));
        for (long s = 0; s < ns; s++) {
            if (costas_out) {
                costas_out[2 * s] = costas_out[2 * s + 1] = 0;
                if (s > 0 && d.order) {
                    const double step = 6.283185307179586 / d.order, dp = (double)cr[s].ph_start - (double)cr[s - 1].ph_end;
                    costas_out[2 * s] = dp - std::nearbyint(dp / step) * step;
                    costas_out[2 * s + 1] = (double)cr[s].fr_start - (double)cr[s - 1].fr_end;
                }
            }
            if (mm_out) {
                mm_out[s] = 0;
                if (s > 0) {
                    const double tref = (double)mr[s - 1].u_final + (double)mr[s - 1].mu_final;
                    const int sk = std::min(std::max(mr[s].skip, 0), 3);
                    mm_out[s] = ((double)mr[s].head_u[sk] + (double)mr[s].head_mu[sk]) - tref;
                }
            }
        }
        *nseg_out = ns;
        *seg_len = d.last_L;
    });
}
int b200_demod_debug_repair_merge(b200_demod *h, int enable)
{
    return guarded([&] {
        B200_REQUIRE(h, B200_EINVAL, "NULL argument");
        h->d->repair_merge = enable != 0;
    });
}
int b200_demod_debug_shape(b200_demod *h, int range_tiles, int seg_len, int keep_front)
{
    return guarded([&] {
        B200_REQUIRE(range_tiles >= 0, B200_EINVAL, "range_tiles %d: a range has at least one tile (0 = the production rule)", range_tiles);
        B200_REQUIRE(seg_len == 0 || (seg_len >= 4096 && seg_len <= 16384 && seg_len % 16 == 0), B200_EINVAL,
                     "seg_len %d: the loop kernels take a multiple of 16 in [4096, 16384] (0 = the production rule)", seg_len);
        B200_REQUIRE(h, B200_EINVAL, "NULL argument");
        Demod &d = *h->d;
        B200_REQUIRE(!(keep_front && d.cfg.keep_stages), B200_EINVAL,
                     "keep_front copies the production front kernel's output, which a keep_stages handle does not run");
        if (keep_front && !d.fir_dump.p) {
            DeviceGuard g(d.cfg.device);
            d.fir_dump.alloc(d.max_work);
        }
        d.dbg_range_tiles = range_tiles;
        d.dbg_seg_len = seg_len;
        d.keep_front = keep_front != 0;
    });
}
int b200_demod_debug_loop_cycles(unsigned long long *out, int cap)
{
    return guarded([&] {
        B200_REQUIRE(out && cap >= LC_SLOTS, B200_EINVAL, "need room for %d counters", (int)LC_SLOTS);
#ifdef B200_LOOP_CYCLES
        B200_CUDA(cudaDeviceSynchronize());
        B200_CUDA(cudaMemcpyFromSymbol(out, g_loop_cycles, sizeof(unsigned long long) * LC_SLOTS));
        const unsigned long long zero[LC_SLOTS] = {};
        B200_CUDA(cudaMemcpyToSymbol(g_loop_cycles, zero, sizeof(zero)));
#else
        B200_REQUIRE(false, B200_EUNSUPPORTED, "this library was built without -DB200_LOOP_CYCLES");
#endif
    });
}
int b200_demod_reset(b200_demod *h)
{
    return guarded([&] {
        B200_REQUIRE(h, B200_EINVAL, "NULL argument");
        h->d->reset();
    });
}
int b200_demod_prefetch_iq(b200_demod *h, const void *host_iq, long n)
{
    return guarded([&] {
        B200_REQUIRE(h && host_iq, B200_EINVAL, "NULL argument");
        h->d->prefetch_host(host_iq, n);
    });
}
int b200_demod_last_timing(b200_demod *h, float *ms, int n)
{
    return guarded([&] {
        B200_REQUIRE(h && ms && n >= 4, B200_EINVAL, "need room for 4 floats");
        ms[1] = h->d->t_agcfir;
        ms[2] = h->d->t_costas;
        ms[3] = h->d->t_mm;
        ms[0] = ms[1] + ms[2] + ms[3];
    });
}
int b200_demod_get_stats(b200_demod *h, b200_demod_stats *out)
{
    return guarded([&] {
        B200_REQUIRE(h && out, B200_EINVAL, "NULL argument");
        h->d->stats(out);
    });
}
int b200_demod_get_taps(b200_demod *h, float *rrc_out, int rrc_cap, float *bank_out)
{
    return guarded([&] {
        B200_REQUIRE(h && rrc_out, B200_EINVAL, "NULL argument");
        B200_REQUIRE((int)h->d->rrc.size() <= rrc_cap, B200_ESTATE, "rrc_out too small");
        memcpy(rrc_out, h->d->rrc.data(), h->d->rrc.size() * sizeof(float));
        if (bank_out)
            memcpy(bank_out, h->d->bank.data(), 128 * 8 * sizeof(float));
    });
}
}

// exposed to api_chain.cu
namespace b200
{
Demod *demod_of(b200_demod *h) { return h->d; }
}
