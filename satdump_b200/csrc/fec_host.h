// Host side of the decoder. Fec is the handle of ONE stream: the soft FIFO, the frame output, the counters every kind reports, and the
// one Decoder that turns the FIFO's soft bytes into frames. The convolutional decoders (Conv, api_fec.cu) mirror
// MetOpAHRPTDecoderModule::process (plugins/noaa_metop_support/metop/module_metop_ahrpt_decoder.cpp:34-90) and
// CCSDSConvConcatDecoderModule::process (src-core/pipeline/modules/ccsds/module_ccsds_conv_concat_decoder.cpp:140-200); the others live in
// api_ldpc.cu, api_turbo.cu, api_dump.cu, api_meteor.cu and api_hrpt.cu; the stages they share are Deframer, FrameStage and Viterbi.
#pragma once
#include "fec.cuh"
#include "walk.cuh"
#include "host_common.h"
#include <memory>
#include <vector>

namespace b200
{

struct DefrEvent { long pos; int state; int pad; };
class Fec;
struct Deframer;
struct FrameStage;

// One decoder kind behind the handle: its kernels consume the soft FIFO of Fec. Every push of the decoders other than Conv reads begin
// -> the decoder's kernels -> keep_soft_tail -> end (or the decoder's own timing).
struct Decoder
{
    long tail_seen = -1;              // FIFO bytes left by the last pass (a second process() without new bytes changes nothing)
    long base_off = 0;                // stream offset of the FIFO's first byte
    long last_nf = 0;                 // records of the last push
    bool keeps_frame_bits = false;    // noaa_gac_decoder, dmsp_rtd_decoder: the stream bit that completed each frame (b200_fec_frame_bits)
    float t_ms[6]{};                  // device ms of the last push's stages, as the decoder's timing getter lists them

    virtual ~Decoder() = default;
    virtual void process(Fec &f) = 0;
    virtual void reset(Fec &f);       // a new stream: the FIFO, its stream offset, the frame bits (the counters carry over)
    virtual void stats(b200_fec_stats *) {} // what the decoder reports beyond the counters of Fec (Fec::stats fills the defaults)
    virtual const Deframer *deframer() const { return nullptr; } // the bit FIFO b200_fec_debug_bits reads

    bool begin(Fec &f, int F);        // false when there is nothing to do: no new bytes, or fewer than F in the FIFO
    void end(Fec &f);                 // waits for the push, checks it, and puts its device time ev[0] .. ev[1] in t_vit
};

// One bit FIFO and the k_deframe machine that walks it (BPSK_CCSDS_Deframer). The FIFO starts with 32 zero bits, the machine's empty
// shifter; a decoder appends its bits at fifo_bits and calls deframe().
struct Deframer
{
    DevBuf<uint32_t> fifo;
    DevBuf<DefrState> dstate;         // [0] the machine, [1] the machine at the last mark() (the MetOp rollback reads it)
    PinnedBuf<DefrState> h_dstate;    // mirror of [0]
    DevBuf<DefrEvent> devents;        // the state changes of the last deframe()
    PinnedBuf<DefrEvent> h_events;
    long fifo_bits = 32, max_events = 0;
    int n_events = 0;                 // ... their number
    int state_now = 2, st_synced = 12, cadu_size = 0;
    uint32_t asm_sync = 0;

    // the machine and the frame counters of Fec at a point a pass may have to roll back to
    struct Mark { DefrState h_dstate; long fifo_bits, out_frames, total_frames, rs_corrected, rs_failed; int state_now; };

    static long frames_cap(long max_new_bits, int cadu_size) { return max_new_bits / cadu_size + 4; } // frames one push can complete
    // room for max_new_bits new bits a push; the whole FIFO is cleared
    void alloc(Fec &f, long max_new_bits, int cadu_size, uint32_t asm_sync, int st_synced);
    void start(Fec &f, size_t clear_bytes); // a new stream: the machine and the FIFO's first clear_bytes
    void compact(Fec &f);             // keeps from the open frame's payload, or the 31 bits of shifter history
    Mark mark(const Fec &f);
    void rewind(Fec &f, const Mark &m);
    int deframe(Fec &f, FrameStage &fs, long new_bits); // walks the new bits, and the frame stage on the frames found: their number
};

// What runs behind a deframer: the RS tables, the frame list, k_frames and the rs_usecheck filter into the frame output of Fec, and the
// RS statistics. meteor_lrpt_decoder and metop_dump_decoder run their own frame kernels on its tables and results.
struct FrameStage
{
    long max_frames = 0;              // frames one push can bring
    int smem = 0;                     // dynamic shared memory of k_frames
    DevBuf<FrameRec> frames;          // the deframer's frames of the last push
    DevBuf<uint8_t> frames_tmp;       // rs_usecheck: the frames in front of the filter
    DevBuf<int> rs_err, frame_dst;    // RS result of every codeword; rs_usecheck: destination index of every frame
    DevBuf<int> counters;             // [0] frames found, [1] deframer state changes, [2] frames rs_usecheck keeps
    DevBuf<RsTables> tables;
    PinnedBuf<int> h_counters, h_rs_err;

    void alloc(Fec &f, long max_frames, int rs_i, bool usecheck); // frames of f.cadu_bytes with rs_i codewords each
    void run(Fec &f, const uint32_t *fifo, int nf); // k_frames (and rs_usecheck) on the nf frames of the list, into frames_out
    // rs_usecheck on nf frames at `in` whose RS results are in rs_err: the frames whose rs_i codewords all decoded, in order, to `out`;
    // their number arrives in h_counters.p[2] (valid after the stream synchronises)
    void usecheck(Fec &f, const uint8_t *in, int nf, int rs_i, uint8_t *out);
    void count_rs(Fec &f, int nf, int rs_i); // rs_corrected / rs_failed of the nf frames in h_rs_err
};

// The parallel Viterbi decoder (r=1/2 or MetOp's r=3/4, k=7): its storage and the state it carries from push to push
struct Viterbi
{
    VitGeom geom{};
    int tb_blocks = 1;
    DevBuf<uint2> dec;                // decisions of every chunk
    DevBuf<uint32_t> chunk_bits;      // decoded bits, geom.bit_words per chunk
    DevBuf<int> start_state;
    DevBuf<int> redo_list;            // chunks decoded again because their speculated start state was wrong (+ the chunks whose BER check follows)
    DevBuf<VitRec> rec;
    DevBuf<TbEdge> tb_edges;
    DevBuf<int> tb_list;              // [0] count of chunks redone serially in the last launch, [1..] their indices
    PinnedBuf<VitRec> h_rec;
    std::vector<int> h_redo, h_redo_ber, h_start;
    VitHyp hyp{0, 0, 0};
    int main_next_start = -1, enc_state = 0;
    int spec_steps = 0, tb_overlap = TB_OVERLAP; // speculation window and warm-up rows of the parallel chainback (adapt to the channel)
    int spec_clean = 0, tb_clean = 0; // consecutive launches without misses (the windows shrink back slowly)
    long start_redone = 0, tb_serial_total = 0; // chunks decoded again from a corrected start state / chained back serially

    void alloc(Fec &f, const VitGeom &g, long max_chunks); // g's chunk, F and BER settings; the strides follow
    int decode_pass(Fec &f, const int8_t *src, long c, int nrange, long out_base, int n, const int *qlist, int nber, const int *ber_list);
    void decode_range(Fec &f, const int8_t *src, long c, int n, long out_base, int max_rounds);
    // Viterbi27 (meteor_lrpt_decoder): the n chunks at src (geom.chunk bytes apart, already rotated) decoded as consecutive calls of ONE
    // chained CCDecoder and its BER encoder, with no lock machine. Chunk q's bits land in chunk_bits[q], its BER error count in ber_errors[q].
    void chained(Fec &f, const int8_t *src, long n, int *ber_errors);
    void stats(b200_fec_stats *o) const;
};
// the last of the `nbits` hard bits of chunk q of chunk_bits (NRZ-M decodes the next bit against it)
int last_raw_bit(Fec &f, const uint32_t *chunk_bits, int bit_words, long q, int nbits);

// The decoders driven by a correlator (ccsds_ldpc_decoder, ccsds_turbo_decoder, metop_dump_decoder, meteor_lrpt_decoder in api_ldpc.cu,
// api_turbo.cu, api_dump.cu, api_meteor.cu): the correlator scores every position of the soft FIFO, k_frame_walk (walk.cuh) goes
// o -> o + pos + F over its windows, the frames are decoded, and the FIFO keeps the bytes behind the walk's next window. Their process()
// reads begin -> correlate -> walk -> walked -> decode -> keep_soft_tail -> timings -> finish.
struct Correlated : Decoder
{
    DevBuf<float> score, bval;        // the correlator's score at every position, the maxima of 32-position blocks
    DevBuf<int> bidx;                 // ... and their positions
    DevBuf<unsigned char> bsync;      // the correlator's table index at every position
    DevBuf<WalkFrame> frames;         // the walk's records
    DevBuf<WalkOut> walk;
    PinnedBuf<WalkOut> h_walk;
    PinnedBuf<WalkFrame> h_frames;    // records of the last push (offsets made absolute)
    long max_frames = 0, resyncs = 0;
    int lock = 0;
    float cor = 0.f;

    void reset(Fec &f) override;      // ... and the lock
    void stats(b200_fec_stats *o) override; // correlator_lock, correlator_corr and ldpc_resyncs

    void alloc(long positions, long frames_cap); // the correlator's outputs for `positions` scores, the walk's records
    int walked(cudaStream_t stream);  // waits for the walk; its frame count
    void finish(int nf, long soft_have); // records made absolute, resyncs, lock and cor of the last frame, the next pass's start
};
std::unique_ptr<Decoder> conv_decoder(Fec &f);      // metop_ahrpt_decoder, ccsds_conv_concat_decoder, ccsds_simple_psk_decoder (api_fec.cu)
std::unique_ptr<Decoder> ldpc_decoder(Fec &f);
std::unique_ptr<Decoder> turbo_decoder(Fec &f);
std::unique_ptr<Decoder> dump_decoder(Fec &f);
std::unique_ptr<Decoder> meteor_decoder(Fec &f);
std::unique_ptr<Decoder> sync_walk_decoder(Fec &f); // noaa_hrpt_decoder, meteor_hrpt_decoder, dmsp_rtd_decoder (api_hrpt.cu)
std::unique_ptr<Decoder> bit_stage_decoder(Fec &f); // aqua_db_decoder, noaa_gac_decoder (api_hrpt.cu)
std::unique_ptr<Decoder> xband_decoder(Fec &f);     // meteor_xband_decoder (api_hrpt.cu)

class Fec
{
  public:
    explicit Fec(const b200_fec_cfg &cfg);
    ~Fec();
    // soft FIFO: the producer writes `n` bytes at append_ptr() then calls commit(n)
    int8_t *append_ptr() { return softbuf.p + soft_have; }
    long append_room() const { return (long)softbuf.n - soft_have; }
    void commit(long n) { soft_have += n; total_soft += n; }
    void push(const int8_t *src, long n, cudaMemcpyKind kind); // append n soft bytes from host or device memory, then process()
    void process(); // decode every complete chunk in the FIFO
    long pull(uint8_t *host_out, long cap);
    void stats(b200_fec_stats *o);
    void reset(); // back to the state of a freshly created decoder (new stream), keeping all allocations

    // The decoder's constructor calls this once its settings are checked and the device is selected: the stream and events, the soft
    // FIFO of max_soft + 2F bytes with keep_soft_tail's scratch, and the frame output for `frames_per_push` frames of cadu_bytes a push.
    void open(int F, long frames_per_push);
    void keep_soft_tail(long used); // keeps the FIFO's bytes behind the `used` ones

    b200_fec_cfg cfg;
    int chunk = 0;      // soft bytes a stream reader of the decoder hands over at a time (b200_fec_chunk_size)
    int cadu_bytes = 0; // bytes of one output unit
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[2]{}, evm[2]{}, evf[2]{};
    float t_vit = 0, t_frames = 0, t_vit_main = 0; // ms of the last process(): whole decoder stage, deframe+RS, k_vit_acs3 alone
    long last_main_chunks = 0;                      // chunks those k_vit_acs3 launches decoded

    std::unique_ptr<Decoder> decoder; // always set
    template <class D> D &decoder_as(const char *what) // the decoder as a D, or B200_EINVAL with `what`
    {
        D *d = dynamic_cast<D *>(decoder.get());
        B200_REQUIRE(d, B200_EINVAL, "%s", what);
        return *d;
    }
    // noaa_gac_decoder / dmsp_rtd_decoder: the stream bit that completed each frame waiting in frames_out, and each frame of the last pull
    std::vector<long> done_bits, pulled_bits;
    void note_frame_bits(long out0, const std::vector<long> &bits); // the bits of the frames a push wrote from frames_out index out0
    long frame_bits(long *out, long cap);

    DevBuf<int8_t> softbuf, soft_tmp; // soft_tmp: keep_soft_tail's scratch (2F bytes)
    DevBuf<uint8_t> frames_out;
    long soft_have = 0;
    long out_frames = 0;                 // frames waiting in frames_out
    long last_bits0 = 0, last_nbits = 0; // range of the decoder's bit FIFO that the last process() appended (debug)
    // statistics
    int rs_avg = 0; // (errors[0] + .. + errors[3]) / 4 of the last frame with rs_i = 4 (meteor_lrpt_decoder's "rs_avg")
    long total_soft = 0, total_chunks = 0, total_bits = 0, total_frames = 0, rs_corrected = 0, rs_failed = 0, replays = 0, launches = 0;
};

// the CCSDS sequence (x^8+x^7+x^5+x^3+1 from all ones), one bit per entry as derand_ccsds_soft applies it to soft bytes (255 entries)
void ccsds_pn_bits(unsigned char *pn);

} // namespace b200

// the handle of the C ABI (each decoder's file defines the entry points that read its records)
struct b200_fec
{
    b200::Fec *f;
};
