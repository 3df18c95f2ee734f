// Host-side C++ mirror of the reference's module layer for the hot path, written above the C ABI (include/b200dsp.h).
//
//   PskDemodStage   <-> satdump::pipeline::demod::PSKDemodModule        (src-core/pipeline/modules/demod/module_psk_demod.cpp)
//                       satdump::pipeline::demod::PMDemodModule         (src-core/pipeline/modules/demod/module_pm_demod.cpp), module id "pm_demod"
//   FecStage        <-> metop::MetOpAHRPTDecoderModule                   (plugins/noaa_metop_support/metop/module_metop_ahrpt_decoder.cpp)
//                       satdump::pipeline::ccsds::CCSDSConvConcatDecoderModule (src-core/pipeline/modules/ccsds/module_ccsds_conv_concat_decoder.cpp)
//   FusedStage      both, with the soft stream kept in HBM
//   run_two_stage() <-> Pipeline::run's two-module streaming mode        (src-core/pipeline/pipeline_run.cpp:44-117)
//
// Same module ids, parameter names, data planes (file / byte FIFO), output formats (.soft = raw int8, .cadu = raw frames) and
// error behaviour (bad / missing parameters throw from the constructor like satdump_exception; process() is void and blocking;
// stop() may be called from another thread; stats are atomics). plugin/b200_dsp_support.cpp wraps these classes into genuine
// satdump::pipeline::ProcessingModule subclasses when built inside a SatDump tree. No CPU fallback anywhere.
#pragma once
#include "../../include/b200dsp.h"
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

namespace b200host
{

// thrown from constructors / init for bad parameters (the plugin shim rethrows it as satdump_exception)
struct ModuleError : std::runtime_error { using std::runtime_error::runtime_error; };

// Pipeline-JSON parameters: name -> JSON scalar as text ("6e6", "qpsk", "true"). The plugin shim fills it from nlohmann::json.
class Params
{
    std::map<std::string, std::string> kv;
  public:
    Params() = default;
    Params(std::initializer_list<std::pair<const std::string, std::string>> l) : kv(l) {}
    void set(const std::string &k, const std::string &v) { kv[k] = v; }
    bool has(const std::string &k) const { return kv.count(k) > 0; }
    std::string str(const std::string &k) const;                 // throws ModuleError when absent
    std::string str(const std::string &k, const std::string &d) const { return has(k) ? kv.at(k) : d; }
    double num(const std::string &k) const;
    double num(const std::string &k, double d) const { return has(k) ? num(k) : d; }
    bool flag(const std::string &k, bool d) const;
};

// Blocking byte FIFO with the semantics of dsp::RingBuffer<uint8_t> (src-core/common/dsp/buffer.h:185-400): read/write block until
// all bytes moved, return -1 once the corresponding side was stopped.
class ByteFifo
{
    std::vector<uint8_t> buf;
    size_t head = 0, fill = 0;
    std::mutex m;
    std::condition_variable can_read, can_write;
    bool stop_r = false, stop_w = false;
  public:
    explicit ByteFifo(size_t capacity = 1000000) : buf(capacity) {}
    int write(const uint8_t *data, int len);
    int read(uint8_t *data, int len);
    int readable();
    void stopReader();
    void stopWriter();
};

enum class DataType { FILE, STREAM }; // DATA_FILE / DATA_STREAM of module.h:48-55

class StageBase
{
  public:
    virtual ~StageBase() = default;
    virtual void init() {}
    virtual void process() = 0; // blocking
    virtual void stop() { should_stop = true; }
    virtual std::string getID() const = 0;
    virtual std::string getOutput() const { return output_file; }
    void setInputType(DataType t) { in_type = t; }
    void setOutputType(DataType t) { out_type = t; }
    std::shared_ptr<ByteFifo> input_fifo, output_fifo;
    std::atomic<bool> input_active{false};
  protected:
    StageBase(std::string in, std::string out_hint, Params p) : input_file(std::move(in)), output_hint(std::move(out_hint)), params(std::move(p)) {}
    std::string input_file, output_hint, output_file;
    Params params;
    DataType in_type = DataType::FILE, out_type = DataType::FILE;
    std::atomic<bool> should_stop{false};
};

// psk_demod: required samplerate, constellation, rrc_alpha, pll_bw (+ symbolrate); optional as in SURVEY.md App. B.
// Options whose blocks are not part of this build (has_carrier, doppler, dump_intermediate) raise ModuleError instead of silently doing
// something else. module_id "pm_demod": PMDemodModule's parameter set (pll_bw = the carrier PLL's, costas_bw, pll_max_offset,
// resample_after_pll, subcarrier_offset), soft = clamp(real * 100), stats key "freq" = the carrier PLL's frequency. module_id
// "fsk_demod": FSKDemodModule's parameter set (rrc_alpha required, its own clock defaults; basic_shaping refused by name).
// "terra_db_demod": TerraDBDemodModule's fixed chain (BPSK loops at twice "symbolrate"); a working rate below 1.1 samples per half-symbol
// is refused by name.
class PskDemodStage : public StageBase
{
  public:
    PskDemodStage(std::string input_file, std::string output_file_hint, Params parameters, std::string module_id = "psk_demod");
    ~PskDemodStage() override;
    void init() override;
    void process() override;
    std::string getID() const override { return id; }
    // getModuleStats() keys of PSKDemodModule (module_psk_demod.cpp:238-246)
    std::atomic<double> progress{0}, freq{0};
    std::atomic<float> snr{0}, peak_snr{0}; // M2M4SNREstimator over the recovered symbols (module_psk_demod.cpp:190-194)
    std::atomic<uint64_t> filesize{0};
    b200_demod_cfg cfg{};
    long batch_samples = 1 << 24;
  private:
    std::string id;
    b200_demod *h = nullptr;
    bool is_bpsk = false;
    size_t data_offset = 0; // first sample of the input file (behind a ZIQ header)
};

// metop_ahrpt_decoder (params viterbi_outsync_after, viterbi_ber_thresold) and ccsds_conv_concat_decoder (App. B list).
class FecStage : public StageBase
{
  public:
    FecStage(const std::string &module_id, std::string input_file, std::string output_file_hint, Params parameters);
    ~FecStage() override;
    void init() override;
    void process() override;
    std::string getID() const override { return id; }
    // getModuleStats() keys: deframer_lock, viterbi_ber, viterbi_lock, rs_avg (module_metop_ahrpt_decoder.cpp:92-104)
    std::atomic<int> viterbi_lock{0}, deframer_state{2};
    std::atomic<float> viterbi_ber{10.f};
    // ccsds_ldpc_decoder: correlator_lock, correlator_corr, ldpc_corr (module_ccsds_ldpc_decoder.cpp:279-295); deframer_state above.
    // ccsds_turbo_decoder: correlator_lock, correlator_corr and crc_lock, what its window shows (module_ccsds_turbo_decoder.cpp:259-290)
    // metop_dump_decoder: "lock_state" = correlator_lock (module_metop_dump_decoder.cpp:84-90)
    std::atomic<int> correlator_lock{0}, ldpc_corr{0};
    std::atomic<float> correlator_corr{0.f};
    std::atomic<int> crc_lock{0};
    // meteor_lrpt_decoder: "rs_avg" of the last frame; m2x_mode 0: correlator_lock, viterbi_ber (module_meteor_lrpt_decoder.cpp:266-289)
    // noaa_hrpt_decoder: "frame_count" = frames_written (words) / 11090; meteor_hrpt_decoder: deframer_state (0 / 2 / 6 / 12), frame_count
    // aqua_db_decoder: deframer_state (2 / 6 / 10) above
    std::atomic<int> rs_avg{0};
    std::atomic<int> viterbi2_lock{0};      // fengyun_ahrpt / _mpt_decoder: "viterbi2_lock" / "viterbi2_ber" (viterbi_* above are viterbi1's)
    std::atomic<float> viterbi2_ber{10.f};
    std::atomic<long> frames_written{0};
    b200_fec_cfg cfg{};
    long batch_soft = 1 << 24;
  private:
    std::string id;
    b200_fec *h = nullptr;
};

// baseband file -> .cadu in one module (soft symbols never leave the GPU). Takes the union of both parameter sets.
class FusedStage : public StageBase
{
  public:
    FusedStage(const std::string &decoder_id, std::string input_file, std::string output_file_hint, Params demod_params, Params decoder_params);
    ~FusedStage() override;
    void init() override;
    void process() override;
    std::string getID() const override { return "b200_psk_" + dec_id; }
    std::atomic<long> frames_written{0};
    std::atomic<int> correlator_lock{0}; // the decoder's correlator lock ("lock_state" of metop_dump_decoder / ccsds_ldpc_decoder)
    std::atomic<int> deframer_state{0};  // meteor_hrpt_decoder: its deframer's state (0 / 2 / 6 / 12)
    std::atomic<double> progress{0};
    long batch_samples = 1 << 26;
  private:
    std::string dec_id;
    Params dparams;
    b200_demod_cfg dcfg{};
    b200_fec_cfg fcfg{};
    b200_chain *h = nullptr;
    size_t data_offset = 0; // first sample of the input file (behind a ZIQ header)
};

b200_demod_cfg demod_cfg_from_params(const Params &p, bool &is_bpsk, const std::string &module_id = "psk_demod");
b200_demod_cfg pm_demod_cfg_from_params(const Params &p, bool &is_bpsk);
b200_fec_cfg fec_cfg_from_params(const std::string &module_id, const Params &p);

// Two modules as two threads joined by a 1 000 000-byte FIFO, like Pipeline::run (pipeline_run.cpp:72-104) minus its 1 s polling.
void run_two_stage(StageBase &m1, StageBase &m2);

} // namespace b200host
