// Host side of the decoder: owns the soft FIFO, the lock machine and the deframer/RS bookkeeping of ONE stream and
// launches the kernels of fec.cuh. Mirrors MetOpAHRPTDecoderModule::process
// (plugins/noaa_metop_support/metop/module_metop_ahrpt_decoder.cpp:34-90) and CCSDSConvConcatDecoderModule::process
// (src-core/pipeline/modules/ccsds/module_ccsds_conv_concat_decoder.cpp:140-200).
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

// A decoder that replaces the Viterbi path (Fec::framed): its own kernels consume the soft FIFO of Fec, and the deframer and frame stage
// of the convolutional decoders serve it where it needs them. Every push reads begin -> the decoder's kernels -> keep_soft_tail -> end
// (or the decoder's own timing).
struct Framed
{
    long tail_seen = -1;              // FIFO bytes left by the last pass (a second process() without new bytes changes nothing)
    long base_off = 0;                // stream offset of the FIFO's first byte
    long last_nf = 0;                 // records of the last push
    float t_ms[6]{};                  // device ms of the last push's stages, as the decoder's timing getter lists them

    virtual ~Framed() = default;
    virtual void process(Fec &f) = 0;
    virtual void reset(Fec &f);       // a new stream: the FIFO, its stream offset, the frame bits (the counters carry over)
    virtual void stats(b200_fec_stats *) {}

    bool begin(Fec &f, int F);        // false when there is nothing to do: no new bytes, or fewer than F in the FIFO
    void end(Fec &f);                 // waits for the push, checks it, and puts its device time ev[0] .. ev[1] in t_vit
};

// The decoders driven by a correlator (ccsds_ldpc_decoder, ccsds_turbo_decoder, metop_dump_decoder, meteor_lrpt_decoder in api_ldpc.cu,
// api_turbo.cu, api_dump.cu, api_meteor.cu): the correlator scores every position of the soft FIFO, k_frame_walk (walk.cuh) goes
// o -> o + pos + F over its windows, the frames are decoded, and the FIFO keeps the bytes behind the walk's next window. Their process()
// reads begin -> correlate -> walk -> walked -> decode -> keep_soft_tail -> timings -> finish.
struct Correlated : Framed
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
std::unique_ptr<Framed> ldpc_decoder(Fec &f);
std::unique_ptr<Framed> turbo_decoder(Fec &f);
std::unique_ptr<Framed> dump_decoder(Fec &f);
std::unique_ptr<Framed> meteor_decoder(Fec &f);
std::unique_ptr<Framed> sync_walk_decoder(Fec &f); // noaa_hrpt_decoder, meteor_hrpt_decoder, dmsp_rtd_decoder (api_hrpt.cu)
std::unique_ptr<Framed> bit_stage_decoder(Fec &f); // aqua_db_decoder, noaa_gac_decoder (api_hrpt.cu)
std::unique_ptr<Framed> xband_decoder(Fec &f);     // meteor_xband_decoder (api_hrpt.cu)

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

    b200_fec_cfg cfg;
    VitGeom geom;
    int cadu_bytes = 0, nphases = 0, ph0 = 0, ph1 = 0, nswap = 0, st_synced = 0, spec_steps = 0; // (a Framed decoder sets only what it uses)
    int fr_smem = 0; // dynamic shared memory of k_frames
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[2];
    float t_vit = 0, t_frames = 0, t_vit_main = 0; // ms of the last process(): whole Viterbi stage, deframe+RS, k_vit_acs3 alone
    cudaEvent_t evm[2], evf[2];
    long last_main_chunks = 0;
    void reset();
    // every kind but METOP, CCSDS and SIMPLE: set up by the constructor instead of the Viterbi / deframer storage
    std::unique_ptr<Framed> framed;
    template <class D> D &framed_as(const char *what) // the decoder as a D, or B200_EINVAL with `what`
    {
        D *d = dynamic_cast<D *>(framed.get());
        B200_REQUIRE(d, B200_EINVAL, "%s", what);
        return *d;
    }
    // noaa_gac_decoder / dmsp_rtd_decoder: the stream bit that completed each frame waiting in frames_out, and each frame of the last pull
    std::vector<long> done_bits, pulled_bits;
    void note_frame_bits(long out0, const std::vector<long> &bits); // the bits of the frames a push wrote from frames_out index out0
    long frame_bits(long *out, long cap);

    // device storage
    DevBuf<int8_t> softbuf;
    DevBuf<uint2> dec;
    DevBuf<uint2> idle_dec;
    DevBuf<uint32_t> chunk_bits, fifo;
    DevBuf<int> start_state, rs_err, counters, frame_dst; // frame_dst: destination index of every frame under rs_usecheck
    DevBuf<VitRec> rec;
    DevBuf<TbEdge> tb_edges;
    DevBuf<int> tb_list; // [0] count of chunks redone serially in the last launch, [1..] their indices
    DevBuf<int> redo_list; // chunks decoded again because their speculated start state was wrong (+ the chunks whose BER check follows)
    std::vector<int> h_redo, h_redo_ber, h_start;
    // Viterbi_Depunc (conv_rate 2/3 ... 7/8): the depunctured symbol stream the decoder windows read (leftover of the previous push in
    // front), the lock search's persistent test buffer, per-window count of real tail symbols, and the DepuncXX / ViterbiSlidingBuffer
    // state of viterbi_punc.cpp / depunc.h carried between pushes
    bool punc = false;
    PuncTab ptab{};
    DevBuf<unsigned char> vitbuf, vitbuf_tmp, bdep;
    DevBuf<int> tail_real;
    DevBuf<PuncIdleOut> punc_out;
    PinnedBuf<PuncIdleOut> h_punc;
    std::vector<int> h_tail, h_wcall;
    long in_buffer = 0;       // symbols waiting in vitbuf (ViterbiSlidingBuffer::in_buffer)
    int changing_shift = 0;   // DepuncXX::changing_shift
    bool is_first = false, got_extra = false;
    int buf_value = 128;      // DepuncXX::buf: the last symbol a call held back
    int test_bit_len = 0;     // Viterbi_Depunc::test_bit_len
    int pdec_start = -1;      // start state of the chained test decoder (cc_decoder_ber)
    int tb_blocks = 1;
    int tb_overlap = TB_OVERLAP; // warm-up rows of the parallel chainback blocks (adapts to the channel)
    int tb_clean = 0, spec_clean = 0; // consecutive launches without misses (the windows shrink back slowly)
    long tb_serial_total = 0, start_redone = 0; // chunks chained back serially / decoded again from a corrected start state
    DevBuf<VitIdleOut> idle_out;
    DevBuf<VitIdle2Out> idle2_out;
    PinnedBuf<VitIdle2Out> h_idle2;
    DevBuf<DefrState> dstate;
    DevBuf<DefrEvent> devents;
    DevBuf<FrameRec> frames;
    DevBuf<uint8_t> frames_out, frames_tmp;
    DevBuf<RsTables> tables;
    // ccsds_simple_psk_decoder: second deframer (QPSK without NRZ-M runs one on the symbols as they are, one on the 90-degree
    // rotated ones) and the carried registers of the hard-decision stage
    DevBuf<uint32_t> chunk_bits2, fifo2;
    DevBuf<DefrState> dstate2;
    DevBuf<int> slice_carry; // [2][2]: oqpsk_delay register, QPSKDiff's previous symbol (ping-pong by call)
    DefrState h_dstate2{};
    long fifo_bits2 = 32;
    int defr_state2 = 2, slice_par = 0, last_nf = 0;
    // QPSK without NRZ-M runs the second deframer
    bool two_deframers() const { return cfg.kind == B200_FEC_SIMPLE && cfg.constellation == B200_QPSK && !cfg.nrzm; }
    void swap_unit();
    void compact_fifo(bool sync);
    void start_stream(size_t fifo_bytes);
    int last_raw_bit(long q, int nbits);
    void keep_soft_tail(long used);
    void deframe_and_rs(long new_bits);
    void framed_storage(int F, long frames_per_push); // what every Framed decoder needs of the decoder object
    void deframer_storage(long max_new_bits); // the bit FIFO, deframer and frame stage behind a Framed decoder's own stages
    // pinned host mirrors
    PinnedBuf<VitRec> h_rec;
    PinnedBuf<VitIdleOut> h_idle;
    PinnedBuf<int> h_counters;
    PinnedBuf<DefrState> h_dstate;
    PinnedBuf<DefrEvent> h_events;
    PinnedBuf<int> h_rs_err;

    // stream state
    long soft_have = 0, max_chunks = 0, fifo_bits = 32, max_frames_push = 0;
    long swapped = 0; // bpsk_90 / iq_invert: FIFO bytes whose pairs are already swapped
    int vit_state = 0, invalid = 0, main_next_start = -1, enc_state = 0, nrzm_last = 0, nosync_runs = 0;
    VitHyp hyp{0, 0, 0};
    VitIdleState idle_st{-1, 0};
    float last_ber = 10.f;
    int defr_state_now = 2;
    int rs_avg = 0; // (errors[0] + .. + errors[3]) / 4 of the last frame with rs_i = 4 (meteor_lrpt_decoder's "rs_avg")
    long out_frames = 0; // frames waiting in frames_out
    long last_bits0 = 0, last_nbits = 0; // FIFO range of the bits appended by the last process() (debug)
    // statistics
    long total_soft = 0, total_chunks = 0, total_bits = 0, total_frames = 0, rs_corrected = 0, rs_failed = 0, replays = 0, launches = 0;

  private:
    // the main deframer and the frame counters at a point a pass may have to roll back to
    struct Mark { DefrState h_dstate; long fifo_bits, out_frames, total_frames, rs_corrected, rs_failed; int defr_state_now; };
    Mark mark();
    void rewind(const Mark &m);
    void decode_simple(long nch);
    void decode_conv(long nch);
};

// Viterbi27 (meteor_lrpt_decoder): the n chunks at src (geom.chunk bytes apart, already rotated) decoded as consecutive calls of ONE chained
// CCDecoder and its BER encoder, with no lock machine. Chunk q's bits land in chunk_bits[q], its BER error count in ber_errors[q].
void viterbi_chained(Fec &f, const int8_t *src, long n, int *ber_errors);
// rs_usecheck on nf frames of cadu_bytes at `in` whose RS results are in f.rs_err: the frames whose rs_i codewords all decoded, in order,
// to `out`; their number arrives in f.h_counters.p[2] (valid after the stream synchronises)
void rs_usecheck_compact(Fec &f, const uint8_t *in, int nf, int rs_i, uint8_t *out);

void build_rs_tables(RsTables &T);
// the CCSDS sequence (x^8+x^7+x^5+x^3+1 from all ones), one bit per entry as derand_ccsds_soft applies it to soft bytes (255 entries)
void ccsds_pn_bits(unsigned char *pn);

} // namespace b200

// the handle of the C ABI (each decoder's file defines the entry points that read its records)
struct b200_fec
{
    b200::Fec *f;
};
