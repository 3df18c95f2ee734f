#include "stream_modules.hpp"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <thread>

namespace b200host
{
// ------------------------------------------------------------------------------------------------ Params
std::string Params::str(const std::string &k) const
{
    auto it = kv.find(k);
    if (it == kv.end())
        throw ModuleError(k + " parameter must be present!");
    return it->second;
}
double Params::num(const std::string &k) const
{
    const std::string s = str(k);
    char *end = nullptr;
    double v = strtod(s.c_str(), &end);
    if (end == s.c_str())
        throw ModuleError("parameter " + k + " is not a number: " + s);
    return v;
}
bool Params::flag(const std::string &k, bool d) const
{
    if (!has(k))
        return d;
    const std::string s = kv.at(k);
    return s == "true" || s == "1";
}

// ------------------------------------------------------------------------------------------------ ByteFifo
int ByteFifo::write(const uint8_t *data, int len)
{
    int done = 0;
    std::unique_lock<std::mutex> lk(m);
    while (done < len) {
        can_write.wait(lk, [&] { return fill < buf.size() || stop_w; });
        if (stop_w)
            return -1;
        size_t n = std::min<size_t>(len - done, buf.size() - fill), tail = (head + fill) % buf.size();
        size_t first = std::min(n, buf.size() - tail);
        memcpy(&buf[tail], data + done, first);
        memcpy(&buf[0], data + done + first, n - first);
        fill += n;
        done += (int)n;
        can_read.notify_one();
    }
    return len;
}
int ByteFifo::read(uint8_t *data, int len)
{
    int done = 0;
    std::unique_lock<std::mutex> lk(m);
    while (done < len) {
        can_read.wait(lk, [&] { return fill > 0 || stop_r; });
        if (stop_r && fill == 0)
            return done > 0 ? done : -1; // end of stream in the middle of a read: hand over what arrived (the caller sees -1 next time)
        size_t n = std::min<size_t>(len - done, fill), first = std::min(n, buf.size() - head);
        memcpy(data + done, &buf[head], first);
        memcpy(data + done + first, &buf[0], n - first);
        head = (head + n) % buf.size();
        fill -= n;
        done += (int)n;
        can_write.notify_one();
    }
    return len;
}
int ByteFifo::readable()
{
    std::lock_guard<std::mutex> lk(m);
    return (int)fill;
}
void ByteFifo::stopReader()
{
    {
        std::lock_guard<std::mutex> lk(m);
        stop_r = true;
    }
    can_read.notify_all();
}
void ByteFifo::stopWriter()
{
    {
        std::lock_guard<std::mutex> lk(m);
        stop_w = true;
    }
    can_write.notify_all();
}

// A junction of the segment-parallel loops that is still inconsistent after the repair rounds means this batch's output may differ
// from the sequential reference around that junction (expected never; b200_demod_stats counts them). The reference's process() has
// no error channel, so this goes where its logger->warn would.
static void warn_unconverged(const b200_demod_stats &st)
{
    if (st.costas_unconverged > 0 || st.mm_unconverged > 0)
        fprintf(stderr, "[b200] warning: %ld Costas / %ld clock-recovery segment junction(s) did not converge in the last batch (after %d repairs so far); "
                        "output around them may deviate from the sequential loop\n", st.costas_unconverged, st.mm_unconverged, st.repairs);
}

// ------------------------------------------------------------------------------------------------ parameter mapping
static void reject(const Params &p, const char *key, const char *why)
{
    if (p.has(key) && p.str(key) != "false" && p.str(key) != "0")
        throw ModuleError(std::string("parameter '") + key + "' is not supported by the B200 path (" + why + "); there is no CPU fallback");
}

// terra_db_demod (module_terra_db_demod.cpp:21-31,84): BaseDemodModule::initb, then RRC(1, final_samplerate, symbolrate * 2, 0.5, 31),
// CostasLoopBlock(0.004, order 2, hz_to_rad(1e6, final_samplerate)), MMClockRecoveryBlock(((float)final_samplerate / (float)symbolrate) / 2,
// pow(0.001, 2) / 4, 0.5, 0.001, 1e-4) and soft = clamp(real * 50): psk_demod's BPSK chain at twice the symbol rate (one soft byte per
// half-symbol), with the working rate chosen for the real symbol rate in BaseDemodModule's window [1.1, 4.0]
static b200_demod_cfg terra_db_demod_cfg_from_params(const Params &p, bool &is_bpsk)
{
    b200_demod_cfg c{};
    if (!p.has("samplerate"))
        throw ModuleError("Samplerate parameter must be present!"); // module_demod_base.cpp:17-20
    c.samplerate = (double)(long)p.num("samplerate");
    if (!p.has("symbolrate"))
        throw ModuleError("Symbolrate parameter must be present!"); // module_demod_base.cpp:26-27
    const double rs = (double)(long)p.num("symbolrate");
    c.symbolrate = 2.0 * rs;
    c.constellation = B200_BPSK;
    is_bpsk = true;
    c.rrc_alpha = 0.5f;
    c.rrc_taps = 31;
    c.pll_bw = 0.004f;
    c.agc_rate = (float)p.num("agc_rate", 1e-2);
    c.clock_gain_omega = (float)(pow(0.001, 2) / 4.0);
    c.clock_mu = 0.5f;
    c.clock_gain_mu = 0.001f;
    c.clock_omega_limit = 0.0001f;
    const std::string fmt = p.str("baseband_format", "cf32");
    if (fmt == "cf32" || fmt == "f32") c.format = B200_CF32;
    else if (fmt == "cs16" || fmt == "s16") c.format = B200_CS16;
    else if (fmt == "cs8" || fmt == "s8") c.format = B200_CS8;
    else if (fmt == "ziq") c.format = -1;
    else throw ModuleError("baseband_format " + fmt + " is not supported by the B200 path (cf32/cs16/cs8, uncompressed ziq)");
    c.dc_block = p.flag("dc_block", false);
    c.freq_shift = (double)(long)p.num("freq_shift", 0);
    c.iq_swap = p.flag("iq_swap", false);
    reject(p, "enable_doppler", "Doppler correction");
    reject(p, "dump_intermediate", "intermediate dump");
    const float min_sps = (float)p.num("min_sps", 0), max_sps = (float)p.num("max_sps", 0);
    c.final_samplerate = b200_demod_final_samplerate(c.samplerate, rs, B200_BPSK, min_sps, max_sps,
                                                     p.has("custom_samplerate") ? (double)(long)p.num("custom_samplerate") : 0.0);
    const double work = c.final_samplerate;
    if (c.final_samplerate == c.samplerate)
        c.final_samplerate = 0;
    else if (!b200_demod_resample_decision(c.samplerate, rs, B200_BPSK, min_sps, max_sps))
        c.front_resample = 2;
    if ((float)c.samplerate / (float)rs < 1.0f) // module_demod_base.cpp:96-105
        throw ModuleError("Your sampling rate is too low! Minimum: " + std::to_string(rs / 1e6) + " Msps");
    // the loops run at half-symbol rate: a working rate inside [1.1, 4.0] samples per symbol can be below 1.1 per half-symbol
    const float half_sps = (float)work / (float)c.symbolrate;
    if (half_sps < 1.1f)
        throw ModuleError("terra_db_demod: samplerate " + std::to_string((long)work) + " gives " + std::to_string(half_sps) +
                          " samples per half-symbol at symbolrate " + std::to_string((long)rs) + "; the loops need at least 1.1");
    c.costas_max_offset = (float)(2.0 * M_PI * (1e6 / work)); // dsp::hz_to_rad(1e6, final_samplerate)
    c.device = (int)p.num("b200_device", 0);
    return c;
}

// fsk_demod (module_fsk_demod.cpp:13-57): required samplerate, symbolrate, rrc_alpha; optional rrc_taps, clock_alpha, clock_gain_omega,
// clock_mu, clock_gain_mu, clock_omega_relative_limit + BaseDemodModule's options, in the constructor's order. The base working window
// [1.1, 4.0] samples per symbol (module_demod_base.h:71-72; the module's own override is commented out)
static b200_demod_cfg fsk_demod_cfg_from_params(const Params &p, bool &is_bpsk)
{
    b200_demod_cfg c{};
    if (!p.has("samplerate"))
        throw ModuleError("Samplerate parameter must be present!"); // module_demod_base.cpp:17-20
    c.samplerate = (double)(long)p.num("samplerate");
    if (!p.has("symbolrate"))
        throw ModuleError("Symbolrate parameter must be present!");
    c.symbolrate = (double)(long)p.num("symbolrate");
    c.constellation = B200_BPSK; // one real symbol, one soft byte each (module_fsk_demod.cpp:133-134)
    is_bpsk = true;
    c.fsk_demod = 1;
    // basic_shaping replaces the RRC by final_sps taps of 0.1 (:75-80); only the 31-tap RRC kernel is built
    reject(p, "basic_shaping", "basic_shaping: the boxcar filter is not built");
    if (!p.has("rrc_alpha"))
        throw ModuleError("RRC Alpha parameter must be present!"); // :21-24
    c.rrc_alpha = (float)p.num("rrc_alpha");
    c.rrc_taps = (int)p.num("rrc_taps", 31);
    c.agc_rate = (float)p.num("agc_rate", 1e-2);
    c.clock_gain_omega = (float)(pow(1.7e-2, 2) / 4.0); // module_fsk_demod.h:28-31
    c.clock_mu = 0.5f;
    c.clock_gain_mu = 1.7e-2f;
    c.clock_omega_limit = 0.005f;
    if (p.has("clock_alpha")) { // :29-35: the float alpha squared (exactly, in double), then rounded to the float member
        const float a = (float)p.num("clock_alpha");
        c.clock_gain_omega = (float)(pow(a, 2) / 4.0);
        c.clock_gain_mu = a;
    }
    c.clock_gain_omega = (float)p.num("clock_gain_omega", c.clock_gain_omega);
    c.clock_mu = (float)p.num("clock_mu", c.clock_mu);
    c.clock_gain_mu = (float)p.num("clock_gain_mu", c.clock_gain_mu);
    c.clock_omega_limit = (float)p.num("clock_omega_relative_limit", c.clock_omega_limit);
    const std::string fmt = p.str("baseband_format", "cf32");
    if (fmt == "cf32" || fmt == "f32") c.format = B200_CF32;
    else if (fmt == "cs16" || fmt == "s16") c.format = B200_CS16;
    else if (fmt == "cs8" || fmt == "s8") c.format = B200_CS8;
    else if (fmt == "ziq") c.format = -1;
    else throw ModuleError("baseband_format " + fmt + " is not supported by the B200 path (cf32/cs16/cs8, uncompressed ziq)");
    c.dc_block = p.flag("dc_block", false);
    c.freq_shift = (double)(long)p.num("freq_shift", 0);
    c.iq_swap = p.flag("iq_swap", false);
    reject(p, "enable_doppler", "Doppler correction");
    reject(p, "dump_intermediate", "intermediate dump");
    const float min_sps = (float)p.num("min_sps", 0), max_sps = (float)p.num("max_sps", 0);
    c.final_samplerate = b200_demod_final_samplerate(c.samplerate, c.symbolrate, B200_BPSK, min_sps, max_sps,
                                                     p.has("custom_samplerate") ? (double)(long)p.num("custom_samplerate") : 0.0);
    if (c.final_samplerate == c.samplerate)
        c.final_samplerate = 0;
    else if (!b200_demod_resample_decision(c.samplerate, c.symbolrate, B200_BPSK, min_sps, max_sps))
        c.front_resample = 2;
    if ((float)c.samplerate / (float)c.symbolrate < 1.0f) // module_demod_base.cpp:96-105
        throw ModuleError("Your sampling rate is too low! Minimum: " +
                          (c.symbolrate > 1e6 ? std::to_string(c.symbolrate / 1e6) + " Msps" : std::to_string(c.symbolrate / 1e3) + " ksps"));
    c.device = (int)p.num("b200_device", 0);
    return c;
}

b200_demod_cfg demod_cfg_from_params(const Params &p, bool &is_bpsk, const std::string &module_id)
{
    if (module_id == "fsk_demod")
        return fsk_demod_cfg_from_params(p, is_bpsk);
    if (module_id == "pm_demod")
        return pm_demod_cfg_from_params(p, is_bpsk);
    if (module_id == "terra_db_demod")
        return terra_db_demod_cfg_from_params(p, is_bpsk);
    b200_demod_cfg c{};
    if (!p.has("samplerate"))
        throw ModuleError("Samplerate parameter must be present!"); // module_demod_base.cpp:17-20
    c.samplerate = (double)(long)p.num("samplerate");
    if (!p.has("symbolrate"))
        throw ModuleError("Symbolrate parameter must be present!");
    c.symbolrate = (double)(long)p.num("symbolrate");
    if (!p.has("constellation"))
        throw ModuleError("Constellation type parameter must be present!"); // module_psk_demod.cpp:18-21
    const std::string con = p.str("constellation");
    if (con == "bpsk") c.constellation = B200_BPSK;
    else if (con == "qpsk") c.constellation = B200_QPSK;
    else if (con == "oqpsk") c.constellation = B200_OQPSK;
    else if (con == "8psk") c.constellation = B200_8PSK;
    else throw ModuleError("unknown constellation " + con);
    is_bpsk = c.constellation == B200_BPSK;
    if (!p.has("rrc_alpha"))
        throw ModuleError("RRC Alpha parameter must be present!");
    c.rrc_alpha = (float)p.num("rrc_alpha");
    c.rrc_taps = (int)p.num("rrc_taps", 31);
    if (!p.has("pll_bw"))
        throw ModuleError("PLL BW parameter must be present!");
    c.pll_bw = (float)p.num("pll_bw");
    c.agc_rate = (float)p.num("agc_rate", 1e-2);
    // module_psk_demod.h:36-39 / module_psk_demod.cpp:36-49
    c.clock_gain_omega = (float)(pow(8.7e-3, 2) / 4.0);
    c.clock_mu = 0.5f;
    c.clock_gain_mu = 8.7e-3f;
    c.clock_omega_limit = 0.005f;
    if (p.has("clock_alpha")) {
        float a = (float)p.num("clock_alpha");
        c.clock_gain_omega = (float)(pow(a, 2) / 4.0);
        c.clock_gain_mu = a;
    }
    c.clock_gain_omega = (float)p.num("clock_gain_omega", c.clock_gain_omega);
    c.clock_mu = (float)p.num("clock_mu", c.clock_mu);
    c.clock_gain_mu = (float)p.num("clock_gain_mu", c.clock_gain_mu);
    c.clock_omega_limit = (float)p.num("clock_omega_relative_limit", c.clock_omega_limit);
    c.costas_max_offset = 1.0f;
    const std::string fmt = p.str("baseband_format", "cf32"); // common/dsp/io/baseband_type.cpp:103-127
    if (fmt == "cf32" || fmt == "f32") c.format = B200_CF32;
    else if (fmt == "cs16" || fmt == "s16") c.format = B200_CS16;
    else if (fmt == "cs8" || fmt == "s8") c.format = B200_CS8;
    else if (fmt == "ziq") c.format = -1; // uncompressed ZIQ: the sample type comes from the file header (resolve_ziq, at init)
    else throw ModuleError("baseband_format " + fmt + " is not supported by the B200 path (cf32/cs16/cs8, uncompressed ziq)");
    c.dc_block = p.flag("dc_block", false); // module_demod_base.cpp:33-34,113-114
    c.freq_shift = (double)(long)p.num("freq_shift", 0); // module_demod_base.cpp:36-37,122-123 (long)
    c.iq_swap = p.flag("iq_swap", false); // module_demod_base.cpp:41-42 -> FileSourceBlock
    c.post_costas_dc = p.flag("post_costas_dc", false); // module_psk_demod.cpp:36-37,127-134
    if (p.flag("has_carrier", false)) { // module_psk_demod.cpp:39-40,93-116
        if (c.constellation != B200_BPSK)
            throw ModuleError("For carrier mode, constellation must be BPSK!");
        if (!p.has("carrier_pll_bw"))
            throw ModuleError("Carrier PLL Bw parameter must be present!");
        c.has_carrier = 1;
        c.carrier_pll_bw = (float)p.num("carrier_pll_bw");
        c.carrier_pll_max_offset = (float)p.num("carrier_pll_max_offset", 3.14);
        c.costas_max_offset = 0.2f; // "the offset in frequency should already be resolved" (:116)
    }
    reject(p, "enable_doppler", "Doppler correction");
    // BaseDemodModule::initb (module_demod_base.cpp:59-87): outside [min_sps, max_sps] the front-end resampler converts to this rate
    if (p.has("clock_recovery")) { // B200 extension (no reference module parameter): "gardner" swaps the clock recovery block
        const std::string cr = p.str("clock_recovery");
        if (cr == "gardner")
            c.clock_recovery = 1;
        else if (cr != "mm")
            throw ModuleError("clock_recovery must be \"mm\" or \"gardner\"");
    }
    c.final_samplerate = b200_demod_final_samplerate(c.samplerate, c.symbolrate, c.constellation, (float)p.num("min_sps", 0), (float)p.num("max_sps", 0),
                                                     p.has("custom_samplerate") ? (double)(long)p.num("custom_samplerate") : 0.0);
    if (c.final_samplerate == c.samplerate)
        c.final_samplerate = 0;
    else if (!b200_demod_resample_decision(c.samplerate, c.symbolrate, c.constellation, (float)p.num("min_sps", 0), (float)p.num("max_sps", 0)))
        c.front_resample = 2; // custom_samplerate with an in-window sps: the reference designs its filters for it but does not resample
    if ((float)c.samplerate / (float)c.symbolrate < 1.0f) // module_demod_base.cpp:96-105
        throw ModuleError("Your sampling rate is too low! Minimum: " +
                          (c.symbolrate > 1e6 ? std::to_string(c.symbolrate / 1e6) + " Msps" : std::to_string(c.symbolrate / 1e3) + " ksps"));
    if (p.has("costas_max_offset")) // Hz -> rad/sample at the working rate (module_psk_demod.cpp:116-118)
        c.costas_max_offset = (float)(2.0 * M_PI * (p.num("costas_max_offset") / (c.final_samplerate > 0 ? c.final_samplerate : c.samplerate)));
    reject(p, "dump_intermediate", "intermediate dump");
    c.device = (int)p.num("b200_device", 0);
    return c;
}

// pm_demod (module_pm_demod.cpp:12-58): required samplerate, symbolrate, pll_bw (the carrier PLL's), rrc_alpha; optional
// resample_after_pll, pll_max_offset, rrc_taps, costas_bw, clock_*, subcarrier_offset + BaseDemodModule's options
b200_demod_cfg pm_demod_cfg_from_params(const Params &p, bool &is_bpsk)
{
    b200_demod_cfg c{};
    if (!p.has("samplerate"))
        throw ModuleError("Samplerate parameter must be present!"); // module_demod_base.cpp:17-20
    c.samplerate = (double)(long)p.num("samplerate");
    if (!p.has("symbolrate"))
        throw ModuleError("Symbolrate parameter must be present!");
    c.symbolrate = (double)(long)p.num("symbolrate");
    c.constellation = B200_BPSK;
    is_bpsk = true;
    c.pm_demod = 1;
    c.pm_resample_after_pll = p.flag("resample_after_pll", false); // module_pm_demod.cpp:18-19
    if (!p.has("pll_bw"))
        throw ModuleError("PLL Bw parameter must be present!"); // :21-24
    c.pm_pll_bw = (float)p.num("pll_bw");
    c.pm_pll_max_offset = (float)p.num("pll_max_offset", 0.5); // :26-27, module_pm_demod.h:29
    if (!p.has("rrc_alpha"))
        throw ModuleError("RRC Alpha parameter must be present!"); // :29-32
    c.rrc_alpha = (float)p.num("rrc_alpha");
    c.rrc_taps = (int)p.num("rrc_taps", 31);
    c.pll_bw = (float)p.num("costas_bw", 0.005); // d_loop_bw (module_pm_demod.h:32, .cpp:37-38)
    c.agc_rate = (float)p.num("agc_rate", 1e-2);
    c.clock_gain_omega = (float)p.num("clock_gain_omega", (float)(pow(0.01, 2) / 4.0)); // module_pm_demod.h:34-37
    c.clock_mu = (float)p.num("clock_mu", 0.5);
    c.clock_gain_mu = (float)p.num("clock_gain_mu", 0.01);
    c.clock_omega_limit = (float)p.num("clock_omega_relative_limit", 0.005);
    c.costas_max_offset = 1.0f;
    c.pm_subcarrier_offset = (double)(uint64_t)p.num("subcarrier_offset", 0); // :52-53
    const std::string fmt = p.str("baseband_format", "cf32");
    if (fmt == "cf32" || fmt == "f32") c.format = B200_CF32;
    else if (fmt == "cs16" || fmt == "s16") c.format = B200_CS16;
    else if (fmt == "cs8" || fmt == "s8") c.format = B200_CS8;
    else if (fmt == "ziq") c.format = -1; // uncompressed ZIQ: the sample type comes from the file header (resolve_ziq, at init)
    else throw ModuleError("baseband_format " + fmt + " is not supported by the B200 path (cf32/cs16/cs8, uncompressed ziq)");
    c.dc_block = p.flag("dc_block", false);
    c.freq_shift = (double)(long)p.num("freq_shift", 0);
    c.iq_swap = p.flag("iq_swap", false);
    reject(p, "enable_doppler", "Doppler correction");
    reject(p, "dump_intermediate", "intermediate dump");
    // MAX_SPS = 10 unless the pipeline gives "max_sps" (module_pm_demod.cpp:56, module_demod_base.cpp:61-64)
    const float min_sps = (float)p.num("min_sps", 0), max_sps = (float)p.num("max_sps", 10.0);
    c.final_samplerate = b200_demod_final_samplerate(c.samplerate, c.symbolrate, c.constellation, min_sps, max_sps,
                                                     p.has("custom_samplerate") ? (double)(long)p.num("custom_samplerate") : 0.0);
    if (c.final_samplerate == c.samplerate)
        c.final_samplerate = 0;
    else if (!b200_demod_resample_decision(c.samplerate, c.symbolrate, c.constellation, min_sps, max_sps))
        c.front_resample = 2;
    if ((float)c.samplerate / (float)c.symbolrate < 1.0f)
        throw ModuleError("Your sampling rate is too low! Minimum: " +
                          (c.symbolrate > 1e6 ? std::to_string(c.symbolrate / 1e6) + " Msps" : std::to_string(c.symbolrate / 1e3) + " ksps"));
    c.device = (int)p.num("b200_device", 0);
    return c;
}

b200_fec_cfg fec_cfg_from_params(const std::string &id, const Params &p)
{
    b200_fec_cfg c{};
    if (id == "metop_dump_decoder") { // module_metop_dump_decoder.cpp:18-23: no parameters
        c.kind = B200_FEC_METOP_DUMP;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_QPSK;
        c.cadu_size = 8192;
        return c;
    }
    if (id == "noaa_hrpt_decoder") { // module_noaa_hrpt_decoder.cpp:14-20: deframer_thresold read with no default; 10-bit words as uint16
        c.kind = B200_FEC_NOAA_HRPT;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_BPSK;
        c.cadu_size = 16; // one output unit = one word
        if (!p.has("deframer_thresold"))
            throw ModuleError("noaa_hrpt_decoder: deframer_thresold is required");
        c.deframer_thresold = (int)p.num("deframer_thresold");
        if (c.deframer_thresold < 0 || c.deframer_thresold > 60) // (a 60-bit window is within 60 of anything: the bound of the library)
            throw ModuleError("noaa_hrpt_decoder: deframer_thresold must be 0..60 (got " + std::to_string(c.deframer_thresold) + ")");
        return c;
    }
    if (id == "noaa_gac_decoder") { // module_noaa_gac_decoder.cpp:17: backward read with no default; 4159-byte frames
        c.kind = B200_FEC_NOAA_GAC;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_BPSK;
        c.cadu_size = 33270;
        if (!p.has("backward"))
            throw ModuleError("noaa_gac_decoder: backward is required");
        c.backward = p.flag("backward", false);
        return c;
    }
    if (id == "dmsp_rtd_decoder") { // module_dmsp_rtd_decoder.cpp:16-24: DMSP_Deframer(150, 2), 19-byte frames
        c.kind = B200_FEC_DMSP_RTD;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_BPSK;
        c.cadu_size = 150;
        return c;
    }
    if (id == "meteor_xband_decoder") { // module_meteor_xband_decoder.cpp:14-32, meteor_xband_types.h: instrument_type "mtvza" | "kmss_bpsk"
        c.kind = B200_FEC_METEOR_XBAND;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_BPSK;
        const std::string t = p.has("instrument_type") ? p.str("instrument_type") : "";
        if (t != "mtvza" && t != "kmss_bpsk")
            throw ModuleError("Invalid METEOR instrument type!");
        c.instrument_type = t == "kmss_bpsk";
        c.cadu_size = c.instrument_type ? 481280 : 3040; // one output unit = one .frm record: 60160 | 380 bytes
        // SoftSymbolReader's hard_symbols path starts from an uninitialised buffer (DESIGN §10.5)
        if (p.flag("hard_symbols", false))
            throw ModuleError("meteor_xband_decoder: hard_symbols input is not supported by the B200 path");
        return c;
    }
    if (id == "fengyun_ahrpt_decoder") { // module_fengyun_ahrpt_decoder.cpp:17-20: the three parameters are read with no default (nlohmann's
        // get<>() on the null a missing key gives throws type_error 302); 1024-byte CADUs
        c.kind = B200_FEC_FENGYUN_AHRPT;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_QPSK;
        c.cadu_size = 8192;
        for (const char *k : {"viterbi_outsync_after", "viterbi_ber_thresold", "invert_second_viterbi"})
            if (!p.has(k))
                throw ModuleError(std::string("fengyun_ahrpt_decoder: ") + k + " is required ([json.exception.type_error.302] type must be " +
                                  (k[0] == 'i' ? "boolean" : "number") + ", but is null)");
        c.outsync_after = (int)p.num("viterbi_outsync_after");
        c.ber_thresold = (float)p.num("viterbi_ber_thresold");
        c.invert_second_viterbi = p.flag("invert_second_viterbi", false);
        return c;
    }
    if (id == "fengyun_mpt_decoder") { // module_fengyun_mpt_decoder.cpp:17-20: the two parameters are read with no default (as
        // fengyun_ahrpt_decoder's); the module has no invert_second_viterbi. 1024-byte CADUs
        c.kind = B200_FEC_FENGYUN_MPT;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_QPSK;
        c.cadu_size = 8192;
        for (const char *k : {"viterbi_outsync_after", "viterbi_ber_thresold"})
            if (!p.has(k))
                throw ModuleError(std::string("fengyun_mpt_decoder: ") + k +
                                  " is required ([json.exception.type_error.302] type must be number, but is null)");
        c.outsync_after = (int)p.num("viterbi_outsync_after");
        c.ber_thresold = (float)p.num("viterbi_ber_thresold");
        return c;
    }
    if (id == "aqua_db_decoder") { // module_aqua_db_decoder.cpp:16-22: no parameters; 1024-byte CADUs (Aqua and Aura DB)
        c.kind = B200_FEC_AQUA_DB;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_QPSK;
        c.cadu_size = 8192;
        return c;
    }
    if (id == "meteor_hrpt_decoder") { // module_meteor_hrpt_decoder.cpp:14-20: no parameters; 1024-byte CADUs
        c.kind = B200_FEC_METEOR_HRPT;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_BPSK;
        c.cadu_size = 8192;
        return c;
    }
    if (id == "meteor_lrpt_decoder") { // module_meteor_lrpt_decoder.cpp:22-49; the library refuses "interleaved" by name
        c.kind = B200_FEC_METEOR_LRPT;
        c.device = (int)p.num("b200_device", 0);
        c.constellation = B200_QPSK;
        c.cadu_size = 8192;
        if (!p.has("diff_decode"))
            throw ModuleError("meteor_lrpt_decoder: diff_decode is required");
        c.diff_decode = p.flag("diff_decode", false);
        c.m2x_mode = p.flag("m2x_mode", false);
        if (c.m2x_mode) {
            if (!p.has("viterbi_outsync_after"))
                throw ModuleError("meteor_lrpt_decoder: viterbi_outsync_after is required with m2x_mode");
            if (!p.has("viterbi_ber_thresold"))
                throw ModuleError("meteor_lrpt_decoder: viterbi_ber_thresold is required with m2x_mode");
            c.outsync_after = (int)p.num("viterbi_outsync_after");
            c.ber_thresold = (float)p.num("viterbi_ber_thresold");
            c.interleaved = p.flag("interleaved", false);
        }
        return c;
    }
    if (id == "ccsds_turbo_decoder") { // module_ccsds_turbo_decoder.cpp:17-36,118-119; the library checks the values (turbo_iters >= 1)
        c.kind = B200_FEC_TURBO;
        c.device = (int)p.num("b200_device", 0);
        if (!p.has("turbo_rate"))
            throw ModuleError("Turbo Rate is required!");
        if (!p.has("turbo_base"))
            throw ModuleError("Turbo Base is required!");
        if (!p.has("turbo_iters"))
            throw ModuleError("Turbo Iters is required!");
        c.turbo_base = (int)p.num("turbo_base");
        c.turbo_iters = (int)p.num("turbo_iters");
        if (!(c.turbo_base == 223 || c.turbo_base == 446 || c.turbo_base == 892 || c.turbo_base == 1115))
            throw ModuleError("Turbo Base must be 223, 446, 892 or 1115!");
        const std::string rate = p.str("turbo_rate");
        if (rate == "1/2") c.turbo_rate = 2;
        else if (rate == "1/3") c.turbo_rate = 3;
        else if (rate == "1/4") c.turbo_rate = 4;
        else if (rate == "1/6") c.turbo_rate = 6;
        else throw ModuleError("Invalid Turbo Rate!");
        c.cadu_size = (c.turbo_base + 4) * 8; // what one output frame holds (ASM + base bytes), written to .cadu (:147)
        return c;
    }
    if (id == "ccsds_ldpc_decoder") { // module_ccsds_ldpc_decoder.cpp:19-124
        c.kind = B200_FEC_LDPC;
        c.device = (int)p.num("b200_device", 0);
        const std::string con = p.str("constellation");
        if (con == "bpsk") c.constellation = B200_BPSK;
        else if (con == "qpsk") c.constellation = B200_QPSK;
        else if (con == "oqpsk") c.constellation = B200_OQPSK;
        else throw ModuleError("CCSDS LDPC Decoder : invalid constellation type!");
        c.derandomize = p.flag("derandomize", true);
        const std::string rate = p.str("ldpc_rate");
        if (rate == "1/2") c.ldpc_rate = 1;
        else if (rate == "2/3") c.ldpc_rate = 2;
        else if (rate == "4/5") c.ldpc_rate = 4;
        else if (rate == "7/8") c.ldpc_rate = 7;
        else throw ModuleError("Invalid LDPC code rate " + rate);
        c.ldpc_block_size = (int)p.num("ldpc_block_size", 0);
        c.ldpc_iterations = (int)p.num("ldpc_iterations");
        c.ldpc2 = p.flag("ldpc2", false);
        // d_internal_stream / d_cadu_size (:33-34): internal_cadu_size is read whenever internal_stream is given
        c.internal_stream = p.flag("internal_stream", false);
        c.internal_cadu_size = p.has("internal_stream") ? (int)p.num("internal_cadu_size") : 0;
        c.asm_sync = p.has("internal_asm") ? (unsigned)std::stoul(p.str("internal_asm"), nullptr, 16) : 0x1ACFFC1D; // (:102-104)
        c.cadu_size = c.internal_stream ? c.internal_cadu_size : 8192; // what one output frame holds
        return c; // ("ccsds": .cadu / .frm output naming, :123, in FecStage::process)
    }
    if (id != "ccsds_simple_psk_decoder") {
        c.outsync_after = (int)p.num("viterbi_outsync_after");
        c.ber_thresold = (float)p.num("viterbi_ber_thresold");
    }
    c.device = (int)p.num("b200_device", 0);
    c.asm_sync = 0x1ACFFC1D;
    if (id == "metop_ahrpt_decoder") {
        c.kind = B200_FEC_METOP;
        c.constellation = B200_QPSK;
        c.cadu_size = 8192;
        return c;
    }
    if (id == "ccsds_simple_psk_decoder") { // module_ccsds_simple_psk_decoder.cpp:19-98
        c.kind = B200_FEC_SIMPLE;
        c.outsync_after = 0;
        c.ber_thresold = 0;
        const std::string con = p.str("constellation");
        if (con == "bpsk") c.constellation = B200_BPSK;
        else if (con == "qpsk") c.constellation = B200_QPSK;
        else throw ModuleError("CCSDS Simple PSK Decoder : invalid constellation type!");
        c.cadu_size = (int)p.num("cadu_size");
        c.qpsk_swap_iq = p.flag("qpsk_swap_iq", false);
        c.qpsk_swap_diff = p.flag("qpsk_swap_diff", true);
        c.oqpsk_delay = p.flag("oqpsk_delay", false);
        if (p.flag("oqpsk_method2", false) || p.flag("oqpsk_method3", false))
            throw ModuleError("oqpsk_method2 / oqpsk_method3 are not supported by the B200 path");
        if (p.flag("hard_symbols", false))
            throw ModuleError("hard_symbols input is not supported by the B200 path");
        c.nrzm = p.flag("nrzm", false);
        c.derandomize = p.flag("derandomize", true);
        c.derand_after_rs = p.flag("derand_after_rs", false);
        c.derand_start = (int)p.num("derand_start", 4);
        c.rs_i = (int)p.num("rs_i");
        c.rs_fill_bytes = (int)p.num("rs_fill_bytes", -1);
        c.rs_dualbasis = p.flag("rs_dualbasis", true);
        const std::string rst = p.str("rs_type", "none");
        if (c.rs_i != 0) {
            if (rst == "rs223") c.rs_type = 0;
            else if (rst == "rs239") c.rs_type = 1;
            else throw ModuleError("CCSDS Simple PSK Decoder : invalid Reed-Solomon type!");
        }
        c.rs_usecheck = p.flag("rs_usecheck", false);
        if (p.has("asm"))
            c.asm_sync = (unsigned)std::stoul(p.str("asm"), nullptr, 16);
        if (p.has("ccsds") && !p.flag("ccsds", true))
            throw ModuleError("ccsds=false (.frm output naming) is not supported by the B200 path");
        return c;
    }
    if (id != "ccsds_conv_concat_decoder")
        throw ModuleError("unknown decoder module " + id);
    c.kind = B200_FEC_CCSDS;
    const std::string con = p.str("constellation"); // module_ccsds_conv_concat_decoder.cpp:38-56
    if (con == "bpsk") c.constellation = B200_BPSK;
    else if (con == "bpsk_90") c.constellation = B200_BPSK_90;
    else if (con == "qpsk") c.constellation = B200_QPSK;
    else if (con == "oqpsk") c.constellation = B200_OQPSK;
    else throw ModuleError("CCSDS Concatenated 1/2 Decoder : invalid constellation type!");
    c.cadu_size = (int)p.num("cadu_size");
    c.nrzm = p.flag("nrzm", false);
    c.derandomize = p.flag("derandomize", true);
    c.derand_after_rs = p.flag("derand_after_rs", false);
    c.derand_start = (int)p.num("derand_start", 4);
    {
        const std::string cr = p.str("conv_rate", "1/2"); // module_ccsds_conv_concat_decoder.cpp:33,99-117
        if (cr == "1/2") c.conv_rate = 0;
        else if (cr == "2/3") c.conv_rate = 2;
        else if (cr == "3/4") c.conv_rate = 3;
        else if (cr == "5/6") c.conv_rate = 5;
        else if (cr == "7/8") c.conv_rate = 7;
        else throw ModuleError("conv_rate " + cr + " is not one of 1/2, 2/3, 3/4, 5/6, 7/8");
    }
    c.rs_i = (int)p.num("rs_i");
    c.rs_fill_bytes = (int)p.num("rs_fill_bytes", -1);
    c.rs_dualbasis = p.flag("rs_dualbasis", true);
    const std::string rst = p.str("rs_type", "none");
    if (c.rs_i != 0) {
        if (rst == "rs223") c.rs_type = 0;
        else if (rst == "rs239") c.rs_type = 1;
        else throw ModuleError("CCSDS Concatenated 1/2 Decoder : invalid Reed-Solomon type!");
    }
    c.rs_usecheck = p.flag("rs_usecheck", false);
    c.iq_invert = p.flag("iq_invert", false);
    if (c.iq_invert)
        throw ModuleError("iq_invert is not supported by the B200 path");
    if (p.has("asm"))
        c.asm_sync = (unsigned)strtoul(p.str("asm").c_str(), nullptr, 16);
    return c;
}

static uint64_t file_size(const std::string &path)
{
    FILE *f = fopen(path.c_str(), "rb");
    if (!f)
        return 0;
    fseek(f, 0, SEEK_END);
    uint64_t n = (uint64_t)ftell(f);
    fclose(f);
    return n;
}
// ZIQ header (src-core/common/ziq.cpp:115-153, docs/pages/ZIQ.md): "ZIQ_", is_compressed (1 byte), bits_per_sample (1 byte), samplerate
// (uint64), annotation length (uint64), annotation; then the samples: int8 / int16 / float32 I,Q pairs, converted exactly like cs8 / cs16 /
// cf32 (ziq.cpp:258-303). Uncompressed files are read here; ZSTD-compressed ones need libzstd, which this build does not link: error.
// Returns the byte offset of the first sample and sets `format`.
static size_t resolve_ziq(const std::string &path, int &format)
{
    FILE *f = fopen(path.c_str(), "rb");
    if (!f)
        throw ModuleError("cannot open " + path);
    unsigned char h[22];
    const size_t got = fread(h, 1, sizeof h, f);
    fclose(f);
    if (got != sizeof h || memcmp(h, "ZIQ_", 4) != 0)
        throw ModuleError("This file is not a valid ZIQ file!"); // ziq.cpp:128-132
    if (h[4])
        throw ModuleError("ZSTD-compressed ZIQ input is not supported by the B200 path (no libzstd in this build): decompress it, or record uncompressed");
    const int bits = h[5];
    if (bits == 8) format = B200_CS8;
    else if (bits == 16) format = B200_CS16;
    else if (bits == 32) format = B200_CF32;
    else throw ModuleError("ZIQ file with " + std::to_string(bits) + " bits per sample");
    uint64_t alen = 0;
    memcpy(&alen, h + 14, 8);
    return (size_t)(22 + alen); // ziq.cpp:178,200: annotation_size + 22
}

static void check(int rc, const char *what)
{
    if (rc != B200_OK)
        throw std::runtime_error(std::string(what) + ": " + b200_last_error());
}

// ------------------------------------------------------------------------------------------------ PskDemodStage
PskDemodStage::PskDemodStage(std::string in, std::string hint, Params p, std::string module_id)
    : StageBase(std::move(in), std::move(hint), std::move(p)), id(std::move(module_id))
{
    if (id != "psk_demod" && id != "pm_demod" && id != "terra_db_demod" && id != "fsk_demod")
        throw ModuleError("unknown demodulator module " + id);
    cfg = demod_cfg_from_params(params, is_bpsk, id);
    batch_samples = (long)params.num("b200_batch_samples", (double)batch_samples);
    cfg.max_batch = batch_samples;
}
PskDemodStage::~PskDemodStage() { b200_demod_destroy(h); }
void PskDemodStage::init()
{
    if (cfg.format < 0) { // baseband_format "ziq"
        if (in_type != DataType::FILE)
            throw ModuleError("ziq input needs a file");
        data_offset = resolve_ziq(input_file, cfg.format);
    }
    h = b200_demod_create(&cfg);
    if (!h)
        throw ModuleError(b200_last_error());
}
void PskDemodStage::process()
{
    if (!h)
        init();
    const int bpsamp = cfg.format == B200_CF32 ? 8 : (cfg.format == B200_CS16 ? 4 : 2);
    std::vector<uint8_t> raw((size_t)batch_samples * bpsamp);
    std::vector<int8_t> soft((size_t)batch_samples * 2 + 4096);
    FILE *fin = nullptr, *fout = nullptr;
    if (in_type == DataType::FILE) {
        fin = fopen(input_file.c_str(), "rb");
        if (!fin)
            throw std::runtime_error("cannot open " + input_file);
        filesize = file_size(input_file);
        if (data_offset)
            fseek(fin, (long)data_offset, SEEK_SET);
    }
    if (out_type == DataType::FILE) {
        output_file = output_hint + ".soft"; // module_psk_demod.cpp:147-151
        fout = fopen(output_file.c_str(), "wb");
    }
    uint64_t done = 0;
    size_t have = 0; // bytes buffered (a batch must hold whole samples and at least 64 of them)
    bool eof = false;
    while (!should_stop && !eof) {
        size_t got;
        if (fin)
            got = fread(raw.data() + have, 1, raw.size() - have, fin);
        else {
            // DATA_STREAM input of raw baseband bytes (the reference feeds a dsp::stream<complex_t> here; a byte FIFO of the
            // configured baseband_format is the C-ABI friendly equivalent)
            int want = (int)std::min<size_t>(raw.size() - have, 1 << 20);
            int r = input_fifo->read(raw.data() + have, want); // a short count = the writer stopped: the stream's last bytes
            got = r < 0 ? 0 : (size_t)r;
        }
        if (got == 0)
            eof = true;
        have += got;
        long ns = (long)(have / bpsamp);
        const long min_batch = cfg.final_samplerate > 0 ? 256 : 64; // the front-end resampler must still yield 64 samples
        if (ns < min_batch || (!eof && have < raw.size() && fin == nullptr && ns < 65536))
            continue;
        check(b200_demod_push_iq(h, raw.data(), ns), "b200_demod_push_iq");
        long n = 0;
        check(b200_demod_pull_soft(h, soft.data(), (long)soft.size(), &n), "b200_demod_pull_soft");
        if (fout)
            fwrite(soft.data(), 1, (size_t)n, fout);
        else if (output_fifo->write((uint8_t *)soft.data(), (int)n) < 0)
            break;
        size_t used = (size_t)ns * bpsamp;
        memmove(raw.data(), raw.data() + used, have - used);
        have -= used;
        done += used;
        progress = filesize ? (double)done / (double)filesize : 0.0;
        b200_demod_stats st;
        if (b200_demod_get_stats(h, &st) == B200_OK) {
            warn_unconverged(st);
            // rad_to_hz(freq, final_samplerate) of the Costas loop (module_psk_demod.cpp:196) / of the carrier PLL (module_pm_demod.cpp:138)
            freq = (cfg.pm_demod ? st.pll_freq : st.costas_freq) * (cfg.final_samplerate > 0 ? cfg.final_samplerate : cfg.samplerate) / (2.0 * M_PI);
            snr = st.snr;
            peak_snr = st.peak_snr;
        }
    }
    if (fin)
        fclose(fin);
    if (fout)
        fclose(fout);
}

// ------------------------------------------------------------------------------------------------ FecStage
// noaa_gac_decoder with backward writes hint + ".frm.tmp" and at the end rewrites ".frm" in reverse frame order, then removes the
// ".tmp" file (module_noaa_gac_decoder.cpp:41-46,113-133); every other decoder writes its output file directly
static std::string frame_file(const b200_fec_cfg &c, const std::string &hint, bool ccsds)
{
    if (c.kind == B200_FEC_NOAA_GAC)
        return hint + (c.backward ? ".frm.tmp" : ".frm");
    if (c.kind == B200_FEC_DMSP_RTD || c.kind == B200_FEC_METEOR_XBAND)
        return hint + ".frm";
    return hint + (c.kind == B200_FEC_NOAA_HRPT ? ".raw16" : (ccsds ? ".cadu" : ".frm"));
}
static void finish_backward(const b200_fec_cfg &c, const std::string &hint)
{
    if (c.kind != B200_FEC_NOAA_GAC || !c.backward)
        return;
    const std::string tmp = hint + ".frm.tmp";
    FILE *in = fopen(tmp.c_str(), "rb");
    FILE *out = fopen((hint + ".frm").c_str(), "wb");
    if (!in || !out)
        throw std::runtime_error("cannot reverse " + tmp);
    std::vector<uint8_t> fr(4159);
    fseek(in, 0, SEEK_END);
    for (long pos = ftell(in) - 4159; pos >= 0; pos -= 4159) {
        fseek(in, pos, SEEK_SET);
        if (fread(fr.data(), 1, fr.size(), in) != fr.size())
            throw std::runtime_error("cannot read " + tmp);
        fwrite(fr.data(), 1, fr.size(), out);
    }
    fclose(in);
    fclose(out);
    remove(tmp.c_str());
}

FecStage::FecStage(const std::string &module_id, std::string in, std::string hint, Params p)
    : StageBase(std::move(in), std::move(hint), std::move(p)), id(module_id)
{
    cfg = fec_cfg_from_params(id, params);
    batch_soft = (long)params.num("b200_batch_soft", (double)batch_soft);
    cfg.max_soft = batch_soft + (1 << 16);
}
FecStage::~FecStage() { b200_fec_destroy(h); }
void FecStage::init()
{
    h = b200_fec_create(&cfg);
    if (!h)
        throw ModuleError(b200_last_error());
}
void FecStage::process()
{
    if (!h)
        init();
    std::vector<int8_t> soft((size_t)batch_soft);
    std::vector<uint8_t> out((size_t)batch_soft / 4 + (1 << 20));
    FILE *fin = nullptr, *fout = nullptr;
    if (in_type == DataType::FILE) {
        fin = fopen(input_file.c_str(), "rb");
        if (!fin)
            throw std::runtime_error("cannot open " + input_file);
    }
    if (out_type == DataType::FILE) {
        const bool ccsds = params.flag("ccsds", true);
        output_file = frame_file(cfg, output_hint, ccsds); // filestream_to_filestream.cpp:27-36, ccsds decoder :131, module_noaa_hrpt_decoder.cpp:20
        fout = fopen(output_file.c_str(), "wb");
        if (cfg.kind == B200_FEC_NOAA_GAC)
            output_file = output_hint + ".frm";
    }
    // dmsp_rtd_decoder's start_timestamp (module_dmsp_rtd_decoder.cpp:36-42,60-66): getValueOrDefault(..., -1)
    const double start_ts = cfg.kind == B200_FEC_DMSP_RTD ? params.num("start_timestamp", -1) : -1;
    FILE *fts = start_ts != -1 ? fopen((output_hint + "_timestamps.txt").c_str(), "wb") : nullptr;
    long ts_reads = 0, ts_last = -1;
    std::vector<long> fbits;
    const int chunk = b200_fec_chunk_size(h);
    while (!should_stop) {
        size_t got;
        if (fin)
            got = fread(soft.data(), 1, soft.size(), fin);
        else {
            // read whole decoder chunks as the reference does (read_data(soft_buffer, BUFFER_SIZE)), several at a time when available
            int avail = input_fifo->readable();
            int want = std::max(chunk, std::min<int>((int)soft.size() / chunk * chunk, avail / chunk * chunk));
            int r = input_fifo->read((uint8_t *)soft.data(), want);
            got = r < 0 ? 0 : (size_t)r;
        }
        if (got == 0)
            break;
        check(b200_fec_push_soft(h, soft.data(), (long)got), "b200_fec_push_soft");
        long nb = 0;
        check(b200_fec_pull_frames(h, out.data(), (long)out.size(), &nb), "b200_fec_pull_frames");
        if (nb > 0) {
            if (fout)
                fwrite(out.data(), 1, (size_t)nb, fout);
            else if (output_fifo->write(out.data(), (int)nb) < 0)
                break;
        }
        if (fts && nb > 0) { // one line per frame: start + 8192 * (the 8192-byte reads that produced frames, up to its own) / 1.024e6
            fbits.resize((size_t)nb / 19 + 1);
            long n = 0;
            check(b200_fec_frame_bits(h, fbits.data(), (long)fbits.size(), &n), "b200_fec_frame_bits");
            for (long k = 0; k < n; k++) {
                const long r = fbits[k] / 8192;
                if (r != ts_last) {
                    ts_reads++;
                    ts_last = r;
                }
                const std::string line = std::to_string(start_ts + double(ts_reads * 8192) / 1.024e6) + "\n";
                fwrite(line.data(), 1, line.size(), fts);
            }
        }
        if (cfg.kind == B200_FEC_TURBO) { // "CRC Check": the CRC of the last frame decoded
            std::vector<b200_turbo_frame> recs(got / 1024 + 4);
            long nrec = 0;
            if (b200_fec_debug_turbo_frames(h, recs.data(), (long)recs.size(), &nrec) == B200_OK && nrec > 0)
                crc_lock = recs[nrec - 1].crc_ok;
        }
        b200_fec_stats st;
        if (b200_fec_get_stats(h, &st) == B200_OK) {
            viterbi_lock = st.viterbi_state;
            viterbi_ber = st.viterbi_ber;
            deframer_state = st.deframer_state;
            frames_written = st.frames_out;
            correlator_lock = st.correlator_lock;
            correlator_corr = st.correlator_corr;
            ldpc_corr = st.ldpc_corr;
            rs_avg = st.rs_avg;
            viterbi2_lock = st.viterbi2_state;
            viterbi2_ber = st.viterbi2_ber;
        }
    }
    if (fin)
        fclose(fin);
    if (fts)
        fclose(fts);
    if (fout) {
        fclose(fout);
        finish_backward(cfg, output_hint);
    }
}

// ------------------------------------------------------------------------------------------------ FusedStage
FusedStage::FusedStage(const std::string &decoder_id, std::string in, std::string hint, Params dp, Params fp)
    : StageBase(std::move(in), std::move(hint), std::move(fp)), dec_id(decoder_id), dparams(std::move(dp))
{
    bool bpsk;
    dcfg = demod_cfg_from_params(dparams, bpsk, dparams.str("b200_demod_module", "psk_demod")); // "pm_demod": PMDemodModule's chain in front
    fcfg = fec_cfg_from_params(dec_id, params);
    if (fcfg.kind == B200_FEC_DMSP_RTD && params.has("start_timestamp")) // (the pipelined chain does not keep the frames' completion bits)
        throw ModuleError("dmsp_rtd_decoder: start_timestamp is not built in the fused chain; run the decoder as its own stage");
    batch_samples = (long)dparams.num("b200_batch_samples", (double)batch_samples);
    dcfg.max_batch = batch_samples;
    fcfg.max_soft = batch_samples + (1 << 20);
    fcfg.device = dcfg.device;
}
FusedStage::~FusedStage() { b200_chain_destroy(h); }
void FusedStage::init()
{
    if (dcfg.format < 0) // baseband_format "ziq"
        data_offset = resolve_ziq(input_file, dcfg.format);
    h = b200_chain_create(&dcfg, &fcfg);
    if (!h)
        throw ModuleError(b200_last_error());
}
void FusedStage::process()
{
    if (!h)
        init();
    const int bpsamp = dcfg.format == B200_CF32 ? 8 : (dcfg.format == B200_CS16 ? 4 : 2);
    std::vector<uint8_t> raw((size_t)batch_samples * bpsamp), out((size_t)batch_samples / 4 + (1 << 20));
    FILE *fin = fopen(input_file.c_str(), "rb");
    if (!fin)
        throw std::runtime_error("cannot open " + input_file);
    const uint64_t fsz = file_size(input_file);
    if (data_offset)
        fseek(fin, (long)data_offset, SEEK_SET);
    output_file = (fcfg.kind == B200_FEC_NOAA_GAC || fcfg.kind == B200_FEC_DMSP_RTD || fcfg.kind == B200_FEC_METEOR_XBAND)
                      ? frame_file(fcfg, output_hint, true)
                                                                                   : output_hint + (fcfg.kind == B200_FEC_NOAA_HRPT ? ".raw16" : ".cadu");
    FILE *fout = fopen(output_file.c_str(), "wb");
    if (fcfg.kind == B200_FEC_NOAA_GAC)
        output_file = output_hint + ".frm";
    uint64_t done = 0;
    size_t have = 0;
    const long min_batch = dcfg.final_samplerate > 0 ? 256 : 64;
    const int cadu_bytes = (fcfg.kind == B200_FEC_METOP) ? 1024 : (fcfg.cadu_size + 7) / 8;
    auto drain = [&]() { // frames of the batches decoded so far (never waits for the one in flight)
        for (;;) {
            long nb = 0;
            check(b200_chain_pull_frames(h, out.data(), (long)out.size(), &nb), "b200_chain_pull_frames");
            if (nb <= 0)
                return;
            fwrite(out.data(), 1, (size_t)nb, fout);
            frames_written += nb / cadu_bytes;
        }
    };
    // decoder one batch behind the demodulator on its own thread / stream, like the reference's two module threads
    check(b200_chain_set_pipelined(h, 1), "b200_chain_set_pipelined");
    while (!should_stop) {
        size_t got = fread(raw.data() + have, 1, raw.size() - have, fin);
        have += got;
        long ns = (long)(have / bpsamp);
        if (ns < min_batch)
            break;
        check(b200_chain_push_iq(h, raw.data(), ns), "b200_chain_push_iq");
        {
            b200_demod_stats dst;
            b200_fec_stats fst;
            if (b200_chain_get_stats(h, &dst, &fst) == B200_OK) {
                warn_unconverged(dst);
                correlator_lock = fst.correlator_lock;
                deframer_state = fst.deframer_state;
            }
        }
        drain();
        size_t used = (size_t)ns * bpsamp;
        memmove(raw.data(), raw.data() + used, have - used);
        have -= used;
        done += used;
        progress = fsz ? (double)done / (double)fsz : 0.0;
        if (got == 0)
            break;
    }
    check(b200_chain_sync(h), "b200_chain_sync");
    drain();
    {
        b200_demod_stats dst;
        b200_fec_stats fst;
        if (b200_chain_get_stats(h, &dst, &fst) == B200_OK)
            deframer_state = fst.deframer_state;
    }
    fclose(fin);
    fclose(fout);
    finish_backward(fcfg, output_hint);
}

// ------------------------------------------------------------------------------------------------ two-module wiring
void run_two_stage(StageBase &m1, StageBase &m2)
{
    auto fifo = std::make_shared<ByteFifo>(1000000); // pipeline_run.cpp:74
    m1.setOutputType(DataType::STREAM);
    m2.setInputType(DataType::STREAM);
    m1.output_fifo = fifo;
    m2.input_fifo = fifo;
    m2.input_active = true;
    m1.init();
    m2.init();
    std::exception_ptr e1, e2;
    std::thread t1([&] { try { m1.process(); } catch (...) { e1 = std::current_exception(); } fifo->stopReader(); });
    std::thread t2([&] { try { m2.process(); } catch (...) { e2 = std::current_exception(); fifo->stopWriter(); } });
    t1.join();
    m2.input_active = false; // the reader drains what is left, then read() returns -1
    t2.join();
    if (e1)
        std::rethrow_exception(e1);
    if (e2)
        std::rethrow_exception(e2);
}

} // namespace b200host
