// SatDump plugin shim: makes the B200 hot path a drop-in for the reference's own modules in UNCHANGED pipeline JSONs.
//
// Built INSIDE a SatDump tree (plugins/b200_dsp_support/, same compiler / flags / headers as libsatdump_core.so — the SatDump <->
// plugin edge is a C++ ABI: src-core/core/plugin.h:10-18, src-core/pipeline/module.h:58-216). It links libb200host.so + libb200dsp.so,
// which are plain C++17 / C ABI and independent of SatDump.
//
//   loader()                          the one symbol SatDump dlsym()s (core/plugin.cpp:15-33)
//   B200DSPSupport::init()            on SatDumpStartedEvent (fired after every plugin registered its modules, init.cpp:163) the
//                                     entries "psk_demod", "pm_demod", "terra_db_demod", "fsk_demod", "metop_ahrpt_decoder", "ccsds_conv_concat_decoder", "ccsds_simple_psk_decoder", "ccsds_ldpc_decoder", "ccsds_turbo_decoder", "metop_dump_decoder", "meteor_lrpt_decoder", "noaa_hrpt_decoder", "meteor_hrpt_decoder", "aqua_db_decoder", "noaa_gac_decoder", "dmsp_rtd_decoder", "meteor_xband_decoder", "fengyun_ahrpt_decoder" and "fengyun_mpt_decoder" of
//                                     satdump::pipeline::modules_registry (module.h:210, looked up first-match by id, module.cpp:129-135)
//                                     get their factory replaced, so existing pipelines instantiate the CUDA modules.
//                                     Set B200_DSP_REGISTER_ONLY=1 to register "<id>_b200" ids instead and leave the originals alone.
//
// In this repository the file is syntax-checked against the genuine headers by __graft_entry__.build() when /root/reference exists;
// satdump_core itself cannot be built in the image (SURVEY.md §0), so the behaviour of the wrapped stages is tested through
// satdump_b200/host (tests/test_gpu_host.py) and the C ABI.
#include "core/exception.h"
#include "core/plugin.h"
#include "logger.h"
#include "pipeline/module.h"
#include "stream_modules.hpp" // satdump_b200/host

#include <cstdlib>
#include <thread>

namespace b200plugin
{
    static b200host::Params to_params(const nlohmann::json &j)
    {
        b200host::Params p;
        for (auto it = j.begin(); it != j.end(); ++it)
        {
            if (it.value().is_string())
                p.set(it.key(), it.value().get<std::string>());
            else if (it.value().is_boolean())
                p.set(it.key(), it.value().get<bool>() ? "true" : "false");
            else if (it.value().is_number())
                p.set(it.key(), it.value().dump()); // the JSON text of the number: std::to_string(double) would print 1.89e-5 as 0.000019
        }
        return p;
    }

    // Bridges SatDump's dsp::RingBuffer<uint8_t> FIFOs to the stage's ByteFifo with two pump threads. (The two FIFO classes
    // have the same blocking semantics; bridging keeps libb200host free of SatDump headers.)
    template <class Stage>
    class WrappedModule : public satdump::pipeline::ProcessingModule
    {
    protected:
        std::shared_ptr<Stage> stage;
        std::string id;

    public:
        WrappedModule(std::string id, std::shared_ptr<Stage> st, std::string in, std::string hint, nlohmann::json params)
            : ProcessingModule(in, hint, params), stage(st), id(id)
        {
        }
        std::vector<satdump::pipeline::ModuleDataType> getInputTypes() override { return {satdump::pipeline::DATA_FILE, satdump::pipeline::DATA_STREAM}; }
        std::vector<satdump::pipeline::ModuleDataType> getOutputTypes() override { return {satdump::pipeline::DATA_FILE, satdump::pipeline::DATA_STREAM}; }
        void init() override
        {
            try
            {
                stage->init();
            }
            catch (const b200host::ModuleError &e)
            {
                throw satdump_exception(e.what());
            }
        }
        void stop() override { stage->stop(); }
        void drawUI(bool) override {} // headless: the CUDA modules have no ImGui panel
        std::string getIDM() override { return id; }
        void process() override
        {
            using namespace satdump::pipeline;
            stage->setInputType(input_data_type == DATA_FILE ? b200host::DataType::FILE : b200host::DataType::STREAM); // (a DSP stream is fed as cf32 bytes)
            stage->setOutputType(output_data_type == DATA_FILE ? b200host::DataType::FILE : b200host::DataType::STREAM);
            std::thread pump_in, pump_out;
            if (input_data_type == DATA_STREAM)
            {
                stage->input_fifo = std::make_shared<b200host::ByteFifo>();
                pump_in = std::thread([this] {
                    std::vector<uint8_t> b(65536);
                    while (input_active.load())
                    {
                        int n = std::min<int>((int)b.size(), std::max(1, input_fifo->getReadable()));
                        if (input_fifo->read(b.data(), n) < 0)
                            break;
                        if (stage->input_fifo->write(b.data(), n) < 0)
                            break;
                    }
                    stage->input_fifo->stopReader();
                });
            }
            if (input_data_type == DATA_DSP_STREAM)
            {
                // dsp::stream<complex_t> (module.h:170; buffer.h:50-107): read() blocks until the writer swapped a buffer in (-1: stopped),
                // readBuf[0..n) are complex floats, flush() hands the buffer back. The stage sees them as a cf32 byte stream.
                stage->input_fifo = std::make_shared<b200host::ByteFifo>();
                pump_in = std::thread([this] {
                    while (input_active.load())
                    {
                        const int n = input_stream->read();
                        if (n < 0)
                            break;
                        const bool ok = n == 0 || stage->input_fifo->write((const uint8_t *)input_stream->readBuf, n * (int)sizeof(complex_t)) >= 0;
                        input_stream->flush();
                        if (!ok)
                            break;
                    }
                    stage->input_fifo->stopReader();
                });
            }
            if (output_data_type == DATA_STREAM)
            {
                stage->output_fifo = std::make_shared<b200host::ByteFifo>();
                pump_out = std::thread([this] {
                    std::vector<uint8_t> b(65536);
                    for (;;)
                    {
                        int n = std::max(1, std::min<int>((int)b.size(), stage->output_fifo->readable()));
                        const int r = stage->output_fifo->read(b.data(), n); // (a short count = the stage stopped writing)
                        if (r < 0)
                            break;
                        if (output_fifo->write(b.data(), r) < 0)
                            break;
                    }
                });
            }
            try
            {
                stage->process();
            }
            catch (const std::exception &e)
            {
                logger->error("b200_dsp_support: %s", e.what()); // process() is void in the reference: runtime problems are logged
                // the stage is gone: release the pump threads (they may sit in a blocking write / read on either FIFO)
                if (stage->input_fifo)
                {
                    stage->input_fifo->stopWriter();
                    stage->input_fifo->stopReader();
                }
                if (input_data_type == DATA_STREAM && input_fifo)
                    input_fifo->stopReader();
                if (input_data_type == DATA_DSP_STREAM && input_stream)
                    input_stream->stopReader();
            }
            d_output_file = stage->getOutput();
            if (stage->output_fifo)
                stage->output_fifo->stopReader();
            if (pump_in.joinable())
                pump_in.join();
            if (pump_out.joinable())
                pump_out.join();
        }
    };

    struct PskDemod : WrappedModule<b200host::PskDemodStage>
    {
        // module_id "psk_demod" (PSKDemodModule) or "pm_demod" (PMDemodModule, module_pm_demod.cpp): same BaseDemodModule data planes and
        // stats keys (progress, snr, peak_snr, freq)
        PskDemod(std::string module_id, std::string in, std::string hint, nlohmann::json p)
            : WrappedModule(module_id, make(module_id, in, hint, p), in, hint, p) {}
        static std::shared_ptr<b200host::PskDemodStage> make(const std::string &module_id, std::string in, std::string hint, const nlohmann::json &p)
        {
            try
            {
                return std::make_shared<b200host::PskDemodStage>(in, hint, to_params(p), module_id);
            }
            catch (const b200host::ModuleError &e)
            {
                throw satdump_exception(e.what());
            }
        }
        // BaseDemodModule: inputs {DATA_FILE, DATA_DSP_STREAM} (+ the byte stream this shim also takes), module_demod_base.cpp:210-212
        std::vector<satdump::pipeline::ModuleDataType> getInputTypes() override
        {
            return {satdump::pipeline::DATA_FILE, satdump::pipeline::DATA_DSP_STREAM, satdump::pipeline::DATA_STREAM};
        }
        void init() override
        {
            if (input_data_type == satdump::pipeline::DATA_DSP_STREAM)
                stage->cfg.format = B200_CF32; // the DSP stream carries complex floats whatever `baseband_format` says (module_demod_base.cpp:96-103)
            WrappedModule::init();
        }
        nlohmann::json getModuleStats() override
        {
            nlohmann::json v; // keys of PSKDemodModule::getModuleStats (module_psk_demod.cpp:238-246)
            if (stage->getID() == "fsk_demod") // FSKDemodModule::getModuleStats (module_fsk_demod.cpp:160-167): no "freq"
            {
                v["progress"] = stage->progress.load();
                v["snr"] = stage->snr.load();
                v["peak_snr"] = stage->peak_snr.load();
                return v;
            }
            if (stage->getID() == "terra_db_demod") // TerraDBDemodModule::getModuleStats (module_terra_db_demod.cpp:138-144)
            {
                v["snr"] = stage->snr.load();
                v["peak_snr"] = stage->peak_snr.load();
                return v;
            }
            v["progress"] = stage->progress.load();
            v["snr"] = stage->snr.load();
            v["peak_snr"] = stage->peak_snr.load();
            v["freq"] = stage->freq.load();
            return v;
        }
    };

    struct Decoder : WrappedModule<b200host::FecStage>
    {
        Decoder(std::string module_id, std::string in, std::string hint, nlohmann::json p)
            : WrappedModule(module_id, make(module_id, in, hint, p), in, hint, p) {}
        static std::shared_ptr<b200host::FecStage> make(const std::string &id, std::string in, std::string hint, const nlohmann::json &p)
        {
            try
            {
                return std::make_shared<b200host::FecStage>(id, in, hint, to_params(p));
            }
            catch (const b200host::ModuleError &e)
            {
                throw satdump_exception(e.what());
            }
        }
        nlohmann::json getModuleStats() override
        {
            nlohmann::json v;
            if (stage->getID() == "ccsds_ldpc_decoder") // CCSDSLDPCDecoderModule::getModuleStats (module_ccsds_ldpc_decoder.cpp:279-295)
            {
                const int ds = stage->deframer_state.load();
                if (stage->cfg.internal_stream)
                {
                    v["deframer_lock"] = ds == 12;
                    v["deframer_state"] = ds == 2 ? "NOSYNC" : (ds == 6 ? "SYNCING" : "SYNCED");
                }
                v["correlator_lock"] = stage->correlator_lock.load() != 0;
                v["correlator_corr"] = stage->correlator_corr.load();
                v["ldpc_corr"] = stage->ldpc_corr.load();
                v["lock_state"] = stage->correlator_lock.load() ? "SYNCED" : "NOSYNC";
                return v;
            }
            if (stage->getID() == "ccsds_turbo_decoder" || stage->getID() == "meteor_xband_decoder") // neither module has getModuleStats:
                return v;                                                                          // ProcessingModule's empty one
            // FengyunAHRPTDecoderModule::getModuleStats (module_fengyun_ahrpt_decoder.cpp:138-152: deframer states 2 / 8 / 16) and
            // FengyunMPTDecoderModule::getModuleStats (module_fengyun_mpt_decoder.cpp:137-153: 2 / 6 / 12)
            if (stage->getID() == "fengyun_ahrpt_decoder" || stage->getID() == "fengyun_mpt_decoder")
            {
                const bool mpt = stage->getID() == "fengyun_mpt_decoder";
                const int ds = stage->deframer_state.load(), v1 = stage->viterbi_lock.load(), v2 = stage->viterbi2_lock.load();
                v["deframer_lock"] = ds == (mpt ? 12 : 16);
                v["viterbi1_ber"] = stage->viterbi_ber.load();
                v["viterbi1_lock"] = v1;
                v["viterbi2_ber"] = stage->viterbi2_ber.load();
                v["viterbi2_lock"] = v2;
                v["rs_avg"] = stage->rs_avg.load();
                v["viterbi1_state"] = v1 == 0 ? "NOSYNC" : "SYNCED";
                v["viterbi2_state"] = v2 == 0 ? "NOSYNC" : "SYNCED";
                v["deframer_state"] = ds == 2 ? "NOSYNC" : (ds == (mpt ? 6 : 8) ? "SYNCING" : "SYNCED");
                return v;
            }
            if (stage->getID() == "metop_dump_decoder") // MetOpDumpDecoderModule::getModuleStats (module_metop_dump_decoder.cpp:84-90)
            {
                v["lock_state"] = stage->correlator_lock.load() ? "SYNCED" : "NOSYNC";
                return v;
            }
            if (stage->getID() == "noaa_hrpt_decoder") // NOAAHRPTDecoderModule::getModuleStats (module_noaa_hrpt_decoder.cpp:47-52)
            {
                v["frame_count"] = stage->frames_written.load() / 11090;
                return v;
            }
            if (stage->getID() == "meteor_hrpt_decoder") // METEORHRPTDecoderModule::getModuleStats (module_meteor_hrpt_decoder.cpp:52-60)
            {
                const int ds = stage->deframer_state.load();
                v["deframer_lock"] = ds == 12;
                v["deframer_state"] = ds == 0 ? "NOSYNC" : (ds == 2 || ds == 6 ? "SYNCING" : "SYNCED");
                v["frame_count"] = stage->frames_written.load();
                return v;
            }
            if (stage->getID() == "noaa_gac_decoder") // NOAAGACDecoderModule::getModuleStats (module_noaa_gac_decoder.cpp:144-150): the
            {                                         // HRPT module's divisor, as the module has it
                v["frame_count"] = stage->frames_written.load() / 11090;
                return v;
            }
            if (stage->getID() == "dmsp_rtd_decoder") // DMSPRTDDecoderModule::getModuleStats (module_dmsp_rtd_decoder.cpp:76-82)
            {
                const int ds = stage->deframer_state.load();
                v["deframer_state"] = ds == 0 ? "NOSYNC" : (ds == 2 ? "SYNCING" : "SYNCED");
                return v;
            }
            if (stage->getID() == "aqua_db_decoder") // AquaDBDecoderModule::getModuleStats (module_aqua_db_decoder.cpp:83-93): SYNCED is state 10
            {
                const int ds = stage->deframer_state.load();
                v["deframer_state"] = ds == 2 ? "NOSYNC" : (ds == 6 ? "SYNCING" : "SYNCED");
                return v;
            }
            if (stage->getID() == "meteor_lrpt_decoder" && !stage->cfg.m2x_mode) // METEORLRPTDecoderModule::getModuleStats (:282-287)
            {
                v["correlator_lock"] = stage->correlator_lock.load() != 0;
                v["viterbi_ber"] = stage->viterbi_ber.load();
                v["rs_avg"] = stage->rs_avg.load();
                v["lock_state"] = stage->correlator_lock.load() ? "SYNCED" : "NOSYNC";
                return v;
            }
            if (stage->getID() == "meteor_lrpt_decoder") // m2x_mode (:271-278): ccsds_conv_concat_decoder's keys below, and rs_avg
                v["rs_avg"] = stage->rs_avg.load();
            // keys of MetOpAHRPTDecoderModule::getModuleStats (module_metop_ahrpt_decoder.cpp:92-104)
            v["deframer_lock"] = stage->deframer_state.load() > 6;
            v["viterbi_ber"] = stage->viterbi_ber.load();
            v["viterbi_lock"] = stage->viterbi_lock.load();
            v["viterbi_state"] = stage->viterbi_lock.load() == 0 ? "NOSYNC" : "SYNCED";
            v["deframer_state"] = stage->deframer_state.load() == 2 ? "NOSYNC" : (stage->deframer_state.load() == 6 ? "SYNCING" : "SYNCED");
            return v;
        }
    };
}

class B200DSPSupport : public satdump::Plugin
{
public:
    std::string getID() { return "b200_dsp_support"; }

    void init()
    {
        const bool register_only = std::getenv("B200_DSP_REGISTER_ONLY") != nullptr;
        if (register_only)
            satdump::eventBus->register_handler<satdump::pipeline::RegisterModulesEvent>(registerHandler);
        else
            satdump::eventBus->register_handler<satdump::SatDumpStartedEvent>(patchHandler);
    }

    using Factory = std::function<std::shared_ptr<satdump::pipeline::ProcessingModule>(std::string, std::string, nlohmann::json)>;
    static Factory factory(const std::string &id)
    {
        if (id == "psk_demod" || id == "pm_demod" || id == "terra_db_demod" || id == "fsk_demod")
            return [id](std::string in, std::string hint, nlohmann::json p) { return std::make_shared<b200plugin::PskDemod>(id, in, hint, p); };
        return [id](std::string in, std::string hint, nlohmann::json p) { return std::make_shared<b200plugin::Decoder>(id, in, hint, p); };
    }

    static void registerHandler(const satdump::pipeline::RegisterModulesEvent &evt)
    {
        for (const char *id : {"psk_demod", "pm_demod", "terra_db_demod", "fsk_demod", "metop_ahrpt_decoder", "ccsds_conv_concat_decoder", "ccsds_simple_psk_decoder", "ccsds_ldpc_decoder",
                               "ccsds_turbo_decoder", "metop_dump_decoder", "meteor_lrpt_decoder", "noaa_hrpt_decoder", "meteor_hrpt_decoder",
                               "aqua_db_decoder", "noaa_gac_decoder", "dmsp_rtd_decoder", "meteor_xband_decoder", "fengyun_ahrpt_decoder",
                               "fengyun_mpt_decoder"})
            evt.modules_registry.push_back({std::string(id) + "_b200", nlohmann::json(), factory(id)});
    }

    static void patchHandler(const satdump::SatDumpStartedEvent &)
    {
        for (auto &e : satdump::pipeline::modules_registry)
            if (e.id == "psk_demod" || e.id == "pm_demod" || e.id == "terra_db_demod" || e.id == "fsk_demod" || e.id == "metop_ahrpt_decoder" || e.id == "ccsds_conv_concat_decoder" || e.id == "ccsds_simple_psk_decoder" ||
                e.id == "ccsds_ldpc_decoder" || e.id == "ccsds_turbo_decoder" || e.id == "metop_dump_decoder" ||
                e.id == "meteor_lrpt_decoder" || e.id == "noaa_hrpt_decoder" || e.id == "meteor_hrpt_decoder" ||
                e.id == "aqua_db_decoder" || e.id == "noaa_gac_decoder" || e.id == "dmsp_rtd_decoder" || e.id == "meteor_xband_decoder" ||
                e.id == "fengyun_ahrpt_decoder" || e.id == "fengyun_mpt_decoder")
            {
                e.inst = factory(e.id);
                logger->info("b200_dsp_support: module " + e.id + " now runs on the B200 path");
            }
    }
};

PLUGIN_LOADER(B200DSPSupport)
