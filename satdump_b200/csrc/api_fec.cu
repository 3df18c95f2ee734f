// C ABI + host driver of the decoder (see include/b200dsp.h, fec_host.h).
#define B200_DEFINE_KERNELS
#include "fec_host.h"
#include <algorithm>
#include <cmath>

namespace b200
{

// one step of the CCSDS randomiser (LFSR h(x) = x^8+x^7+x^5+x^3+1): the bit it outputs
static int pn_step(uint8_t &reg)
{
    const int out = reg >> 7;
    const uint8_t nb = ((reg >> 7) ^ (reg >> 4) ^ (reg >> 2) ^ reg) & 1;
    reg = (uint8_t)((reg << 1) | nb);
    return out;
}

// GF(256) tables exactly as libcorrect builds them (libs/correct/reed-solomon/field.h:26-62: log[1] ends up 255, log[0] = 0),
// CCSDS dual-basis maps (GF(2)-linear, generated from the images of the unit vectors) and the CCSDS randomiser bytes
// (LFSR h(x) = x^8+x^7+x^5+x^3+1 from all ones).
static void build_rs_tables(RsTables &T)
{
    memset(&T, 0, sizeof(T));
    unsigned e = 1;
    T.exp[0] = 1;
    T.log[0] = 0;
    for (int i = 1; i < 512; i++) {
        e <<= 1;
        if (e > 255)
            e ^= 0x187;
        T.exp[i] = (uint8_t)e;
        if (i < 256)
            T.log[e] = (uint8_t)i;
    }
    static const uint8_t img[8] = {0x7B, 0xAF, 0x99, 0xFA, 0x86, 0xEC, 0xEF, 0x8D};
    for (int v = 0; v < 256; v++) {
        uint8_t r = 0;
        for (int b = 0; b < 8; b++)
            if (v >> b & 1)
                r ^= img[b];
        T.to_dual[v] = r;
    }
    for (int v = 0; v < 256; v++)
        T.from_dual[T.to_dual[v]] = (uint8_t)v;
    uint8_t reg = 0xFF;
    for (int i = 0; i < 255; i++) {
        uint8_t byte = 0;
        for (int k = 0; k < 8; k++)
            byte = (uint8_t)((byte << 1) | pn_step(reg));
        T.pn[i] = byte;
    }
}

void ccsds_pn_bits(unsigned char *pn)
{
    uint8_t reg = 0xFF;
    for (int i = 0; i < 255; i++)
        pn[i] = (unsigned char)pn_step(reg);
}

// meteor_lrpt_decoder with m2x_mode (module_meteor_lrpt_decoder.cpp:29-43, 103-197) is ccsds_conv_concat_decoder with constellation
// "oqpsk" (Viterbi1_2 over 8192-byte calls, phases 0 and 90, the IQ-swap check), NRZ-M bits when diff_decode, BPSK_CCSDS_Deframer(8192),
// the derandomiser from byte 4 before RS, RS223 I=4 in the conventional basis and only the frames whose four codewords decode written:
// that configuration, run as kind CCSDS. Every other configuration passes unchanged.
static b200_fec_cfg meteor_m2x_as_ccsds(const b200_fec_cfg &c)
{
    if (c.kind != B200_FEC_METEOR_LRPT || !c.m2x_mode)
        return c;
    B200_REQUIRE(!c.interleaved, B200_EUNSUPPORTED,
                 "meteor_lrpt_decoder: \"interleaved\" is not built: the reference's interleaved reader never delivers a sample (its input "
                 "function always reports failure), so there is no behaviour to reproduce");
    b200_fec_cfg r = c;
    r.kind = B200_FEC_CCSDS;
    r.constellation = B200_OQPSK;
    r.cadu_size = 8192;
    r.conv_rate = 0;
    r.nrzm = c.diff_decode != 0;
    r.derandomize = 1;
    r.derand_after_rs = 0;
    r.derand_start = 4;
    r.rs_i = 4;
    r.rs_dualbasis = 0;
    r.rs_fill_bytes = -1;
    r.rs_usecheck = 1;
    r.rs_type = 0;
    r.iq_invert = 0;
    r.asm_sync = 0x1ACFFC1D;
    return r;
}

// Most deframer state changes (k_deframe's event list) a walk over `max_bits` FIFO bits can record. Every NOSYNC -> SYNCING change
// opens a frame whose cadu_size - 32 payload bits the walk skips before it tests again, and at most two changes follow it (SYNCING ->
// SYNCED -> NOSYNC, or SYNCING -> NOSYNC); the state a push starts in adds at most two more. A noisy stream that loses and finds the
// ASM every few frames stays within this, at any push size.
static long defr_event_cap(long max_bits, int cadu_size)
{
    return 3 * (max_bits / std::max(1, cadu_size - 32) + 2);
}

Fec::Fec(const b200_fec_cfg &in) : cfg(meteor_m2x_as_ccsds(in))
{
    std::unique_ptr<Decoder> (*make)(Fec &) = nullptr;
    switch (cfg.kind) {
    case B200_FEC_METOP: case B200_FEC_CCSDS: case B200_FEC_SIMPLE: make = conv_decoder; break;
    case B200_FEC_LDPC: make = ldpc_decoder; break;
    case B200_FEC_TURBO: make = turbo_decoder; break;
    case B200_FEC_METOP_DUMP: make = dump_decoder; break;
    case B200_FEC_METEOR_LRPT: make = meteor_decoder; break;
    case B200_FEC_NOAA_HRPT: case B200_FEC_METEOR_HRPT: case B200_FEC_DMSP_RTD: make = sync_walk_decoder; break;
    case B200_FEC_AQUA_DB: case B200_FEC_NOAA_GAC: make = bit_stage_decoder; break;
    case B200_FEC_METEOR_XBAND: make = xband_decoder; break;
    case B200_FEC_FENGYUN_AHRPT: case B200_FEC_FENGYUN_MPT: make = fengyun_decoder; break;
    default: B200_REQUIRE(false, B200_EINVAL, "unknown decoder kind %d", cfg.kind);
    }
    B200_REQUIRE(cfg.max_soft >= 65536, B200_EINVAL, "max_soft must be >= 65536");
    decoder = make(*this);
}

struct OutChunk { long soft_chunk; int next_start, enc_tail, invalid_after, state_after; VitIdleState idle_st; };

// metop_ahrpt_decoder, ccsds_conv_concat_decoder (with the punctured rates and meteor_lrpt_decoder's m2x_mode) and
// ccsds_simple_psk_decoder: the lock machine and the Viterbi decoder (SIMPLE: the hard-decision slicer), NRZ-M, the deframer and the
// frame stage over the complete chunks of the soft FIFO
struct Conv : Decoder
{
    const bool metop, simple;
    const bool two;                   // ccsds_simple_psk_decoder QPSK without NRZ-M: a second deframer on the 90-degree rotated symbols
    int nphases = 1, ph0 = 0, ph1 = 0, nswap = 1; // the lock search's hypotheses
    long max_chunks = 0;              // chunks (punctured: decoder windows) one push can bring
    Viterbi vit;                      // (not allocated for SIMPLE)
    Deframer defr, defr2;             // the main deframer; the second one of `two`, run first
    FrameStage fs;                    // (the two deframers share it)
    // the lock machine
    int vit_state = 0, invalid = 0, nrzm_last = 0, nosync_runs = 0;
    VitIdleState idle_st{-1, 0};
    float last_ber = 10.f;
    long swapped = 0;                 // bpsk_90 / iq_invert: FIFO bytes whose pairs are already swapped
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
    // ccsds_simple_psk_decoder: the hard bits of every chunk (slice_words per chunk) for the main and the second deframer, and the
    // carried registers of the hard-decision stage
    int slice_words = 0, slice_par = 0;
    DevBuf<uint32_t> slice_bits, slice_bits2;
    DevBuf<int> slice_carry; // [2][2]: oqpsk_delay register, QPSKDiff's previous symbol (ping-pong by call)

    explicit Conv(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
    void stats(b200_fec_stats *o) override;
    const Deframer *deframer() const override { return &defr; }
    void viterbi_segment(Fec &f, long c0, long nch, std::vector<OutChunk> &outs);
    void punc_segment(Fec &f, long c0, long ncalls, std::vector<OutChunk> &outs);
    void decode_conv(Fec &f, long nch);
    void decode_simple(Fec &f, long nch);
};

Conv::Conv(Fec &f)
    : metop(f.cfg.kind == B200_FEC_METOP), simple(f.cfg.kind == B200_FEC_SIMPLE),
      two(simple && f.cfg.constellation == B200_QPSK && !f.cfg.nrzm)
{
    const b200_fec_cfg c = f.cfg;
    b200_fec_cfg &cfg = f.cfg;
    VitGeom geom{};
    int st_synced = 12;
    if (!metop) {
        B200_REQUIRE(c.cadu_size >= 64 && c.cadu_size <= 65536, B200_EINVAL, "cadu_size out of range");
        B200_REQUIRE(c.cadu_size % 8 == 0, B200_EINVAL, "cadu_size must be a multiple of 8 (frame padding is not built)");
        B200_REQUIRE(c.rs_i >= 0 && c.rs_i <= RS_MAX_I, B200_EINVAL, "rs_i out of range (0..%d)", RS_MAX_I);
        B200_REQUIRE(c.rs_i == 0 || c.cadu_size / 8 >= 4 + 255 * c.rs_i, B200_EINVAL, "cadu_size too small for rs_i interleaved codewords");
        B200_REQUIRE(c.rs_fill_bytes <= 0, B200_EINVAL, "rs_fill_bytes (shortened codes) is not built");
        B200_REQUIRE(c.rs_fill_bytes >= -1, B200_EINVAL, "rs_fill_bytes must be -1 (none) or >= 0 (got %d)", c.rs_fill_bytes);
        B200_REQUIRE(!c.derandomize || c.derand_start >= 0, B200_EINVAL, "derand_start must be >= 0 (got %d)", c.derand_start);
        if (cfg.asm_sync == 0)
            cfg.asm_sync = 0x1ACFFC1D;
    }
    if (metop) {
        // module_metop_ahrpt_decoder.cpp:10,17-25: 16384-byte chunks, r=3/4, phases {0,90}, deframer SYNCED threshold 18, RS223 I=4
        geom.rate34 = 1;
        geom.chunk = 8192 * 2;
        geom.F = geom.chunk * 3 / 4;
        cfg.cadu_size = 8192;
        cfg.rs_i = 4;
        cfg.rs_dualbasis = 1;
        cfg.rs_type = 0;
        cfg.derandomize = 1;
        cfg.derand_after_rs = 0;
        cfg.derand_start = 4;
        cfg.rs_usecheck = 0;
        cfg.nrzm = 0;
        cfg.asm_sync = 0x1ACFFC1D;
        nphases = 2; ph0 = 0; ph1 = 1; nswap = 1;
        st_synced = 18;
        vit.spec_steps = VIT_SPEC_STEPS_34;
    } else if (simple) {
        // module_ccsds_simple_psk_decoder.cpp:19-98: one loop iteration = cadu_size soft bytes -> cadu_size bits
        B200_REQUIRE(c.constellation == B200_BPSK || c.constellation == B200_QPSK, B200_EINVAL, "CCSDS Simple PSK Decoder : invalid constellation type!");
        geom.chunk = c.cadu_size;
        geom.F = c.cadu_size;
    } else {
        // module_ccsds_conv_concat_decoder.cpp:16-131
        geom.chunk = std::max(c.cadu_size, 8192);
        B200_REQUIRE(geom.chunk % 2 == 0, B200_EINVAL, "chunk size must be even");
        geom.F = geom.chunk / 2;
        B200_REQUIRE(c.conv_rate == 0 || c.conv_rate == 2 || c.conv_rate == 3 || c.conv_rate == 5 || c.conv_rate == 7, B200_EINVAL,
                     "conv_rate must be 0 (1/2), 2 (2/3), 3 (3/4), 5 (5/6) or 7 (7/8)");
        if (c.conv_rate) {
            // Viterbi_Depunc(depunc, ber, outsync, buffer_size, phases, oqpsk) (module_ccsds_conv_concat_decoder.cpp:108-117): one module call =
            // buffer_size soft symbols; the decoder works on windows of vit_bufsize = buffer_size DEPUNCTURED symbols (frame buffer_size / 2 bits)
            punc = true;
            geom.raw = 1;
            static const PuncTab tabs[4] = {{3, 4, 3.5f, {1, 2, 1}, {0, 0, 0}, {0, 1, 3, 4}},                                       // depunc.h: Depunc23
                                            {4, 6, 5.0f, {1, 2, 1, 2}, {0, 0, 0, 0}, {0, 1, 3, 4, 6}},                                // Depunc34
                                            {6, 10, 8.0f, {1, 2, 1, 2, 2, 2}, {0, 0, 0, 0, 1, 0}, {0, 1, 3, 4, 6, 8, 10}},             // Depunc56
                                            {8, 14, 10.0f, {1, 2, 2, 2, 1, 2, 2, 2}, {0, 0, 0, 0, 0, 0, 1, 0}, {0, 1, 3, 5, 7, 8, 10, 12, 14}}}; // Depunc78
            ptab = tabs[c.conv_rate == 2 ? 0 : (c.conv_rate == 3 ? 1 : (c.conv_rate == 5 ? 2 : 3))];
        }
        if (c.constellation == B200_BPSK) { nphases = 1; ph0 = 0; ph1 = 0; }
        else if (c.constellation == B200_BPSK_90) { nphases = 1; ph0 = 1; ph1 = 1; }
        else if (c.constellation == B200_QPSK || c.constellation == B200_OQPSK) { nphases = 2; ph0 = 0; ph1 = 1; }
        else B200_REQUIRE(false, B200_EINVAL, "CCSDS Concatenated 1/2 Decoder : invalid constellation type!");
        nswap = c.constellation == B200_OQPSK ? 2 : 1;
        vit.spec_steps = VIT_SPEC_STEPS_12;
    }
    f.chunk = geom.chunk;
    f.cadu_bytes = (cfg.cadu_size + 7) / 8;
    check_device(c.device);
    DeviceGuard g(c.device);
    max_chunks = c.max_soft / geom.chunk + 2;
    if (punc) { // windows per push: the calls' symbols times Q / P, plus the leftover of the push before
        const long max_sym = (c.max_soft / geom.chunk + 2) * (long)geom.chunk * ptab.Q / ptab.P + 2L * geom.chunk + 64;
        max_chunks = max_sym / geom.chunk + 2;
        vitbuf.alloc((size_t)max_sym + geom.chunk + 64);
        vitbuf_tmp.alloc((size_t)2 * geom.chunk + 64);
        bdep.alloc(4 * VIT_TESTLEN);
        tail_real.alloc(max_chunks + 2);
        punc_out.alloc(1);
        h_punc.alloc(1);
    }
    const long max_new_bits = max_chunks * (long)geom.F;
    const long max_frames = Deframer::frames_cap(max_new_bits, cfg.cadu_size);
    f.open(geom.chunk, max_frames);
    if (simple) {
        slice_words = (geom.F + 31) / 32 + 1;
        slice_bits.alloc((size_t)max_chunks * slice_words + 4);
        if (two)
            slice_bits2.alloc(slice_bits.n);
        slice_carry.alloc(4);
    } else {
        vit.alloc(f, geom, max_chunks);
        vit.alloc_lock_search();
    }
    defr.alloc(f, max_new_bits, cfg.cadu_size, cfg.asm_sync, st_synced);
    if (two)
        defr2.alloc(f, max_new_bits, cfg.cadu_size, cfg.asm_sync, st_synced);
    fs.alloc(f, max_frames, cfg.rs_i, cfg.rs_usecheck && cfg.rs_i > 0);
    reset(f);
}

std::unique_ptr<Decoder> conv_decoder(Fec &f) { return std::make_unique<Conv>(f); }

Fec::~Fec()
{
    DeviceGuard g(cfg.device);
    if (stream)
        cudaStreamSynchronize(stream);
    decoder.reset();
    for (cudaEvent_t e : {ev[0], ev[1], evm[0], evm[1], evf[0], evf[1]})
        if (e)
            cudaEventDestroy(e);
    if (stream)
        cudaStreamDestroy(stream);
}

void Fec::push(const int8_t *src, long n, cudaMemcpyKind kind)
{
    B200_REQUIRE(n <= append_room(), B200_ESTATE, "push of %ld soft bytes exceeds the FIFO room %ld (max_soft too small)", n, append_room());
    DeviceGuard g(cfg.device);
    B200_CUDA(cudaMemcpyAsync(append_ptr(), src, n, kind, stream));
    commit(n);
    process();
}

constexpr int WPB = 4; // warps per block of the one-warp-per-chunk kernels (k_vit_acs3 indexes its warps by blockIdx.x * 4)

// An adaptive window follows the channel: many misses in a launch (> 2 % of its chunks) double it up to `cap`; 32 launches in a row
// with almost none (< 0.2 %) halve it back towards `base`. It shrinks slowly because one doubling squares the miss probability, so
// the shorter window would fail again at once on the same channel.
static void adapt_window(int &win, int &clean, double miss_frac, int base, int cap)
{
    if (miss_frac > 0.02) {
        win = std::min(cap, win * 2);
        clean = 0;
    } else if (miss_frac < 0.002 && ++clean >= 32) {
        win = std::max(base, win / 2);
        clean = 0;
    }
}

// One decode pass: ACS, parallel chainback (+ check and serial fallback) and BER counters of `n` chunks of the range of `nrange`
// chunks at c of `src` (all of them, or the ones in `qlist`; the BER check runs on `nber` chunks, or on the ones in `ber_list`). The
// records of the whole range come back to h_rec. Returns the number of chunks chained back serially.
int Viterbi::decode_pass(Fec &f, const int8_t *src, long c, int nrange, long out_base, int n, const int *qlist, int nber, const int *ber_list)
{
    B200_CUDA(cudaEventRecord(f.evm[0], f.stream));
    k_vit_acs3<<<(n + WPB - 1) / WPB, 32 * WPB, 0, f.stream>>>(src, c, n, geom, hyp, start_state.p, dec.p, rec.p, qlist);
    B200_CUDA(cudaEventRecord(f.evm[1], f.stream));
    const long nthr = (long)n * tb_blocks;
    B200_CUDA(cudaMemsetAsync(tb_list.p, 0, sizeof(int), f.stream));
    k_vit_tb<<<(unsigned)((nthr + 127) / 128), 128, 0, f.stream>>>(n, tb_blocks, geom, dec.p, chunk_bits.p, out_base, rec.p, tb_edges.p, qlist, tb_overlap);
    k_vit_tb_check<<<(n + 255) / 256, 256, 0, f.stream>>>(n, tb_blocks, tb_edges.p, tb_list.p, nrange, qlist);
    k_vit_tb_serial<<<(n + 127) / 128, 128, 0, f.stream>>>(tb_list.p, nrange, geom, dec.p, chunk_bits.p, out_base, rec.p); // (threads beyond the list return at once)
    k_vit_ber<<<(nber + WPB - 1) / WPB, 32 * WPB, 0, f.stream>>>(src, c, nber, geom, hyp, chunk_bits.p, out_base, enc_state, rec.p, ber_list);
    f.launches += 5;
    B200_CUDA(cudaMemcpyAsync(h_rec.p, rec.p, sizeof(VitRec) * nrange, cudaMemcpyDeviceToHost, f.stream));
    int tb_redone = 0;
    B200_CUDA(cudaMemcpyAsync(&tb_redone, tb_list.p, sizeof(int), cudaMemcpyDeviceToHost, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream));
    tb_serial_total += tb_redone;
    float ms = 0;
    cudaEventElapsedTime(&ms, f.evm[0], f.evm[1]);
    f.t_vit_main += ms;
    return tb_redone;
}

// Optimistic parallel decode of n consecutive decoder windows (chunks c .. c+n-1 of `src`, geom.chunk bytes apart) into chunk_bits[out_base ..]:
// start-state speculation, one decode pass, and up to `max_rounds` redo rounds for chunks whose speculated start state was wrong. Leaves
// the per-chunk records in h_rec[0 .. n). Each round makes the first inconsistent chunk consistent (its predecessor is not redone), so
// n rounds always settle the range.
void Viterbi::decode_range(Fec &f, const int8_t *src, long c, int n, long out_base, int max_rounds)
{
    B200_CUDA(cudaMemcpyAsync(start_state.p, &main_next_start, sizeof(int), cudaMemcpyHostToDevice, f.stream));
    if (n > 1) {
        k_vit_spec<<<(n - 1 + WPB - 1) / WPB, 32 * WPB, 0, f.stream>>>(src, c, n, geom, hyp, spec_steps, start_state.p);
        f.launches++;
    }
    const int tb_redone = decode_pass(f, src, c, n, out_base, n, nullptr, n, nullptr);
    f.last_main_chunks += n;
    if (n > 64) // the chainback warm-up follows the channel like the speculation window does
        adapt_window(tb_overlap, tb_clean, (double)tb_redone / (double)n, TB_OVERLAP, TB_OVERLAP_MAX);
    // Start states that were speculated wrong (k_vit_spec: common at low SNR, where 768 steps do not always pin the state): those
    // chunks alone are decoded again from the state their predecessor really left. A chunk's end state almost never depends on its
    // start state, so one round normally settles it; a round that changes a successor's start state is followed by another.
    for (int round = 0; round < max_rounds; round++) {
        h_redo.clear();
        for (int i = 1; i < n; i++)
            if (h_rec.p[i].start_used != h_rec.p[i - 1].next_start) {
                h_redo.push_back(i);
                h_start[i] = h_rec.p[i - 1].next_start;
            }
        if (round == 0 && n > 64) // wrong guesses: the survivors of the speculation window had not all merged (low SNR)
            adapt_window(spec_steps, spec_clean, (double)h_redo.size() / (double)n, geom.rate34 ? VIT_SPEC_STEPS_34 : VIT_SPEC_STEPS_12,
                         (geom.F / 32) * 32);
        if (h_redo.empty())
            break;
        const int m = (int)h_redo.size();
        f.replays += m;
        start_redone += m;
        // the BER check of a chunk reads the last test bits of its predecessor: redo it for the successors too
        h_redo_ber = h_redo;
        for (int i : h_redo)
            if (i + 1 < n)
                h_redo_ber.push_back(i + 1);
        std::sort(h_redo_ber.begin(), h_redo_ber.end());
        h_redo_ber.erase(std::unique(h_redo_ber.begin(), h_redo_ber.end()), h_redo_ber.end());
        const int mb = (int)h_redo_ber.size();
        for (int i : h_redo)
            B200_CUDA(cudaMemcpyAsync(start_state.p + i, &h_start[i], sizeof(int), cudaMemcpyHostToDevice, f.stream));
        B200_CUDA(cudaMemcpyAsync(redo_list.p, h_redo.data(), sizeof(int) * m, cudaMemcpyHostToDevice, f.stream));
        B200_CUDA(cudaMemcpyAsync(redo_list.p + n, h_redo_ber.data(), sizeof(int) * mb, cudaMemcpyHostToDevice, f.stream));
        decode_pass(f, src, c, n, out_base, m, redo_list.p, mb, redo_list.p + n);
    }
}

void Viterbi::chained(Fec &f, const int8_t *src, long n, int *ber_errors)
{
    long c = 0;
    while (c < n) {
        const int m = (int)(n - c);
        decode_range(f, src, c, m, c, 6); // (what is still inconsistent after six rounds is decoded again below)
        int accepted = m;
        for (int i = 1; i < m; i++)
            if (h_rec.p[i].start_used != h_rec.p[i - 1].next_start) {
                f.replays++;
                accepted = i;
                break;
            }
        for (int i = 0; i < accepted; i++)
            ber_errors[c + i] = h_rec.p[i].ber_errors;
        main_next_start = h_rec.p[accepted - 1].next_start;
        enc_state = h_rec.p[accepted - 1].enc_tail;
        c += accepted;
    }
}

void Viterbi::alloc_lock_search()
{
    idle_dec.alloc(VIT_TESTLEN + 64);
    idle_out.alloc(1);
    idle2_out.alloc(1);
    h_idle.alloc(1);
    h_idle2.alloc(1);
    B200_CUDA(cudaFuncSetAttribute(k_vit_idle2<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * VIT_IDLE_WARP_BYTES));
    B200_CUDA(cudaFuncSetAttribute(k_vit_idle2<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * VIT_IDLE_WARP_BYTES));
}

const VitIdleOut &Viterbi::lock_search(Fec &f, const int8_t *src, long c, int n, int nswap, int nphases, int ph0, int ph1, VitIdleState st, int mode,
                                       unsigned head)
{
    const float thr = f.cfg.ber_thresold;
    if (mode == VIT_IDLE_R12_EXACT) { // every trial reads the one before it: the serial kernel
        k_vit_idle<VIT_IDLE_R12_EXACT><<<1, 32, 0, f.stream>>>(src, c, n, geom, nswap, nphases, ph0, ph1, thr, st, idle_dec.p, idle_out.p, head);
        f.launches++;
        B200_CUDA(cudaMemcpyAsync(h_idle.p, idle_out.p, sizeof(VitIdleOut), cudaMemcpyDeviceToHost, f.stream));
        B200_CUDA(cudaStreamSynchronize(f.stream));
        return *h_idle.p;
    }
    const bool fy = mode == VIT_IDLE_FY;
    // parallel search first (one warp per hypothesis); it hands over to the serial kernel at the first chunk whose chained 6-bit states
    // its two-pass guess did not reproduce
    const int nh = nswap * nphases * 2;
    auto idle2 = fy ? k_vit_idle2<true> : k_vit_idle2<false>;
    idle2<<<1, 32 * nh, nh * VIT_IDLE_WARP_BYTES, f.stream>>>(src, c, n, geom, nswap, nphases, ph0, ph1, thr, st, idle2_out.p);
    f.launches++;
    B200_CUDA(cudaMemcpyAsync(h_idle2.p, idle2_out.p, sizeof(VitIdle2Out), cudaMemcpyDeviceToHost, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream));
    *h_idle.p = h_idle2.p->o;
    if (h_idle2.p->fallback_chunk >= 0) {
        const long c2 = c + h_idle2.p->fallback_chunk;
        auto idle1 = fy ? k_vit_idle<VIT_IDLE_FY> : k_vit_idle<VIT_IDLE_PLAIN>;
        idle1<<<1, 32, 0, f.stream>>>(src, c2, (int)(n - (c2 - c)), geom, nswap, nphases, ph0, ph1, thr, h_idle2.p->o.st, idle_dec.p, idle_out.p, 0u);
        f.launches++;
        B200_CUDA(cudaMemcpyAsync(h_idle.p, idle_out.p, sizeof(VitIdleOut), cudaMemcpyDeviceToHost, f.stream));
        B200_CUDA(cudaStreamSynchronize(f.stream));
        if (h_idle.p->lock_chunk >= 0)
            h_idle.p->lock_chunk += (int)(c2 - c);
    }
    return *h_idle.p;
}

void Viterbi::alloc(Fec &f, const VitGeom &g, long max_chunks)
{
    geom = g;
    geom.dec_stride = (geom.F + 6 + 7) & ~7;
    geom.bit_words = (geom.F + 31) / 32 + 1;
    tb_blocks = ((geom.F + 31) / 32 + TB_WORDS - 1) / TB_WORDS;
    dec.alloc((size_t)max_chunks * geom.dec_stride);
    chunk_bits.alloc((size_t)max_chunks * geom.bit_words + 4);
    start_state.alloc(max_chunks + 1);
    redo_list.alloc(2 * (size_t)max_chunks + 4); // chunk indices to decode again | chunks whose BER check follows
    h_start.resize(max_chunks + 2);
    rec.alloc(max_chunks + 1);
    h_rec.alloc(max_chunks + 1);
    tb_edges.alloc((size_t)(max_chunks + 1) * tb_blocks);
    tb_list.alloc((size_t)max_chunks + 2); // chunks whose parallel chainback blocks disagreed at an edge (any number: low SNR makes them common)
    rec.zero(f.stream);
}

void FrameStage::usecheck(Fec &f, const uint8_t *in, int nf, int rs_i, uint8_t *out)
{
    k_frames_filter<<<1, 1024, 0, f.stream>>>(rs_err.p, nf, rs_i, frame_dst.p, counters.p + 2);
    k_frames_gather<<<std::min(nf, 132 * 16), 256, 0, f.stream>>>(in, frame_dst.p, nf, f.cadu_bytes, out);
    f.launches += 2;
    B200_CUDA(cudaMemcpyAsync(h_counters.p + 2, counters.p + 2, sizeof(int), cudaMemcpyDeviceToHost, f.stream));
}

// Viterbi over soft chunks [c0, nch): lock search while IDLE, optimistic parallel decode while SYNCED. Decoded chunks land in
// chunk_bits[0 .. nout). Returns per-output-chunk bookkeeping in `outs`.
void Conv::viterbi_segment(Fec &f, long c0, long nch, std::vector<OutChunk> &outs)
{
    outs.clear();
    const VitGeom &geom = vit.geom;
    long c = c0, out_base = 0;
    const float kber = geom.rate34 ? 5.0f : 2.5f;
    while (c < nch) {
        if (vit_state == 0) {
            idle_st.enc_state = vit.enc_state; // ONE chained CCEncoder serves the lock test and the SYNCED BER check (viterbi_3_4.cpp:126,157)
            const VitIdleOut &o = vit.lock_search(f, f.softbuf.p, c, (int)(nch - c), nswap, nphases, ph0, ph1, idle_st, VIT_IDLE_PLAIN);
            idle_st = o.st;
            vit.enc_state = idle_st.enc_state;
            float bb = 10.f;
            for (int i = 0; i < 16; i++)
                bb = std::min(bb, o.bers[i]);
            last_ber = bb;
            if (o.lock_chunk < 0)
                break;
            c += o.lock_chunk;
            vit_state = 1;
            vit.hyp = VitHyp{o.swap, o.phase, o.shift};
            invalid = 0;
            vit.enc_state = idle_st.enc_state;
        }
        const int n = (int)(nch - c);
        vit.decode_range(f, f.softbuf.p, c, n, out_base, 6); // (what is still inconsistent after six rounds is decoded again below)
        const VitRec *rec = vit.h_rec.p;
        int accepted = 0;
        for (int i = 0; i < n; i++) {
            if (i > 0 && rec[i].start_used != rec[i - 1].next_start) {
                f.replays++; // still inconsistent after the redo rounds above: decode again from here with the true state
                break;
            }
            accepted = i + 1;
            const float ber = ((float)rec[i].ber_errors / (float)rec[i].ber_total) * kber;
            last_ber = ber;
            bool lost = false;
            if (ber > f.cfg.ber_thresold) { // viterbi_3_4.cpp:160-169
                invalid++;
                if (invalid > f.cfg.outsync_after) {
                    vit_state = 0;
                    lost = true;
                }
            } else
                invalid = 0;
            outs.push_back(OutChunk{c + i, rec[i].next_start, rec[i].enc_tail, invalid, vit_state, idle_st});
            if (lost)
                break;
        }
        vit.main_next_start = rec[accepted - 1].next_start;
        vit.enc_state = rec[accepted - 1].enc_tail;
        out_base += accepted;
        c += accepted;
    }
}

// ccsds_conv_concat_decoder with conv_rate 2/3 ... 7/8: Viterbi_Depunc::work (viterbi_punc.cpp:53-145) over the module calls [c0, ncalls) of
// the soft FIFO (one call = geom.chunk soft symbols). IDLE: lock search call by call (k_punc_idle). SYNCED: all remaining calls at once -
//   * DepuncXX::depunc_cont of the whole run in closed form into the symbol stream behind the leftover of earlier calls (k_punc_depunc);
//   * ViterbiSlidingBuffer: window w = symbols [w V, w V + V + 12) of that stream is decoded in the first call j whose even-truncated
//     running total T_j exceeds (w + 1) V; what it reads beyond T_j are erasures (the buffer's memset after the previous window; the
//     first window of a call always has its 12 tail symbols, a call makes more than V + 12 symbols at every rate);
//   * the windows go through the same speculative-start ACS / chainback / BER kernels as the fixed-rate decoders (decode_range);
//   * the lock machine is replayed per call on the host: d_ber = BER of the last window decoded in the call.
void Conv::punc_segment(Fec &f, long c0, long ncalls, std::vector<OutChunk> &outs)
{
    outs.clear();
    const int V = vit.geom.chunk, size = vit.geom.chunk;
    const PuncTab &P = ptab;
    auto made = [&](long m) { return (m / P.P) * (long)P.Q + P.cum[m % P.P]; };
    long c = c0, out_base = 0;
    while (c < ncalls) {
        if (vit_state == 0) {
            const VitIdleState st{pdec_start, vit.enc_state};
            k_punc_idle<<<1, 32, 0, f.stream>>>(f.softbuf.p, c, (int)(ncalls - c), size, P, nswap, nphases, ph0, ph1, f.cfg.ber_thresold, st, bdep.p,
                                                vit.idle_dec.p, punc_out.p);
            f.launches++;
            B200_CUDA(cudaMemcpyAsync(h_punc.p, punc_out.p, sizeof(PuncIdleOut), cudaMemcpyDeviceToHost, f.stream));
            B200_CUDA(cudaStreamSynchronize(f.stream));
            const PuncIdleOut &o = *h_punc.p;
            pdec_start = o.st.dec_start;
            vit.enc_state = o.st.enc_state;
            test_bit_len = o.test_bit_len;
            last_ber = o.ber;
            if (o.lock_call < 0)
                break;
            c += o.lock_call;
            vit_state = 1;
            vit.hyp = VitHyp{o.swap, o.phase, 0};
            invalid = 0;
            changing_shift = o.shift; // set_shift (depunc.h)
            is_first = o.shift > P.P - 1;
        }
        const int n = (int)(ncalls - c);
        // depunc_cont of calls c .. c+n-1. A symbol held back by the previous call (got_extra) already sits at vitbuf[in_buffer].
        const int held = got_extra ? 1 : 0;
        const int lead = (!got_extra && is_first) ? 1 : 0; // `buf` emitted in front (its stale value when nothing is held)
        is_first = false;
        const int a0 = changing_shift % P.P;
        const long nsoft = (long)n * size;
        B200_REQUIRE((size_t)(in_buffer + held + lead + made(a0 + nsoft) - made(a0) + 16) <= vitbuf.n, B200_ESTATE, "internal: depunctured stream buffer too small");
        k_punc_depunc<<<(unsigned)((nsoft + 255) / 256), 256, 0, f.stream>>>(f.softbuf.p + c * (long)size, nsoft, vit.hyp, P, a0, lead, buf_value,
                                                                            vitbuf.p + in_buffer + held);
        f.launches++;
        // which call decodes which window, and how much of its 12-symbol tail exists by then
        h_tail.clear();
        h_wcall.clear();
        long w = 0;
        for (int j = 1; j <= n; j++) {
            const long raw = held + lead + made(a0 + (long)j * size) - made(a0);
            const long T = in_buffer + 2 * (raw / 2);
            while (T - w * V > V) {
                h_wcall.push_back(j);
                h_tail.push_back((int)std::min<long>(12, T - (w + 1) * V));
                w++;
            }
        }
        const int nw = (int)w;
        B200_REQUIRE(nw >= 1 && nw <= max_chunks, B200_ESTATE, "internal: window count %d out of range", nw);
        B200_CUDA(cudaMemcpyAsync(tail_real.p, h_tail.data(), sizeof(int) * nw, cudaMemcpyHostToDevice, f.stream));
        vit.geom.tail_real = tail_real.p;
        vit.geom.ber_bits = VIT_TESTLEN;      // cc_encoder_ber.work(output, ...) encodes TEST_BITS_LENGTH bits (viterbi_punc.cpp:124)
        vit.geom.ber_syms = test_bit_len;     // get_ber(vit_buffer, ..., test_bit_len, 5) (:125)
        // the lock machine below accepts windows call by call and has no way back to a window decoded from a wrong start state, so the
        // redo rounds run until every window's start state is its predecessor's next start
        vit.decode_range(f, reinterpret_cast<const int8_t *>(vitbuf.p), 0, nw, out_base, nw);
        const VitRec *rec = vit.h_rec.p;
        // replay the lock machine call by call
        int jacc = n, wacc = nw;
        for (int j = 1, wi = 0; j <= n; j++) {
            int last = -1;
            while (wi < nw && h_wcall[wi] == j)
                last = wi++;
            if (last >= 0)
                last_ber = ((float)rec[last].ber_errors / (float)rec[last].ber_total) * 5.0f;
            if (last_ber > f.cfg.ber_thresold) { // viterbi_punc.cpp:133-141
                invalid++;
                if (invalid > f.cfg.outsync_after) {
                    vit_state = 0;
                    jacc = j;
                    wacc = wi;
                    break;
                }
            } else
                invalid = 0;
        }
        for (int i = 0; i < wacc; i++)
            outs.push_back(OutChunk{c + h_wcall[i] - 1, rec[i].next_start, rec[i].enc_tail, invalid, vit_state, idle_st});
        if (wacc > 0) {
            vit.main_next_start = rec[wacc - 1].next_start;
            vit.enc_state = rec[wacc - 1].enc_tail;
        }
        // what stays in the sliding buffer: the symbols behind the decoded windows up to the last accepted call's total, plus the one
        // that call held back (its value is DepuncXX::buf from now on)
        const long raw = held + lead + made(a0 + (long)jacc * size) - made(a0);
        const long T = in_buffer + 2 * (raw / 2);
        got_extra = raw & 1;
        changing_shift = (int)((a0 + (long)jacc * size) % P.P);
        const long keep0 = (long)wacc * V, keep = T - keep0 + (got_extra ? 1 : 0);
        B200_REQUIRE(keep >= 0 && (size_t)keep <= vitbuf_tmp.n, B200_ESTATE, "internal: sliding buffer leftover %ld", keep);
        if (got_extra) {
            unsigned char hb = 0;
            B200_CUDA(cudaMemcpyAsync(&hb, vitbuf.p + T, 1, cudaMemcpyDeviceToHost, f.stream));
            B200_CUDA(cudaStreamSynchronize(f.stream));
            buf_value = hb;
        }
        if (keep > 0 && keep0 > 0) {
            B200_CUDA(cudaMemcpyAsync(vitbuf_tmp.p, vitbuf.p + keep0, keep, cudaMemcpyDeviceToDevice, f.stream));
            B200_CUDA(cudaMemcpyAsync(vitbuf.p, vitbuf_tmp.p, keep, cudaMemcpyDeviceToDevice, f.stream));
        }
        in_buffer = T - keep0;
        out_base += wacc;
        c += jacc;
    }
}

int Deframer::deframe(Fec &f, FrameStage &fs, long new_bits)
{
    cudaStream_t stream = f.stream;
    const long nbits = fifo_bits + new_bits;
    B200_CUDA(cudaEventRecord(f.evf[0], stream));
    k_deframe<<<1, 32, 0, stream>>>(fifo.p, nbits, cadu_size, st_syncing, st_synced, asm_sync, dstate.p, fs.frames.p, (int)fs.max_frames,
                                   reinterpret_cast<DefrEventDev *>(devents.p), (int)max_events, fs.counters.p);
    f.launches++;
    B200_CUDA(cudaMemcpyAsync(fs.h_counters.p, fs.counters.p, sizeof(int) * 2, cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(h_dstate.p, dstate.p, sizeof(DefrState), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    const int nf = fs.h_counters.p[0];
    n_events = fs.h_counters.p[1];
    B200_REQUIRE(nf <= fs.max_frames, B200_ESTATE, "internal: frame list overflow");
    B200_REQUIRE(n_events <= max_events, B200_ESTATE, "internal: %d deframer state changes in one push, more than the %ld its bits allow", n_events,
                 max_events);
    if (n_events > 0) // (complete at the event synchronise below)
        B200_CUDA(cudaMemcpyAsync(h_events.p, devents.p, sizeof(DefrEvent) * n_events, cudaMemcpyDeviceToHost, stream));
    if (nf > 0)
        fs.run(f, fifo.p, nf);
    B200_CUDA(cudaEventRecord(f.evf[1], stream));
    B200_CUDA(cudaEventSynchronize(f.evf[1]));
    {
        float ms = 0;
        cudaEventElapsedTime(&ms, f.evf[0], f.evf[1]);
        f.t_frames += ms;
    }
    fifo_bits = nbits;
    state_now = h_dstate.p->state;
    return nf;
}

void FrameStage::run(Fec &f, const uint32_t *fifo, int nf)
{
    const b200_fec_cfg &cfg = f.cfg;
    B200_REQUIRE((size_t)(f.out_frames + nf) * f.cadu_bytes <= f.frames_out.n, B200_ESTATE, "frame output buffer full: call pull_frames");
    FrameCfg fc;
    fc.cadu_bytes = f.cadu_bytes;
    fc.cadu_size = cfg.cadu_size;
    fc.derandomize = cfg.derandomize;
    fc.derand_after_rs = cfg.derand_after_rs;
    fc.derand_start = cfg.derand_start;
    fc.rs_i = cfg.rs_i;
    fc.rs_dual = cfg.rs_dualbasis;
    fc.rs_nroots = cfg.rs_type == 1 ? 16 : 32;
    fc.rs_fcr = cfg.rs_type == 1 ? 120 : 112;
    fc.sync = cfg.asm_sync;
    fc.rs_row256 = cfg.rs_fill_bytes == -1;
    const bool filter = cfg.rs_usecheck && cfg.rs_i > 0;
    uint8_t *out = f.frames_out.p + f.out_frames * f.cadu_bytes;
    k_frames<<<std::min(nf, 132 * 8), 256, smem, f.stream>>>(fifo, frames.p, nf, fc, tables.p, filter ? frames_tmp.p : out, rs_err.p);
    f.launches++;
    if (filter)
        usecheck(f, frames_tmp.p, nf, cfg.rs_i, out);
    if (cfg.rs_i > 0)
        B200_CUDA(cudaMemcpyAsync(h_rs_err.p, rs_err.p, sizeof(int) * nf * cfg.rs_i, cudaMemcpyDeviceToHost, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream));
    const int kept = filter ? h_counters.p[2] : nf;
    count_rs(f, nf, cfg.rs_i);
    if (cfg.rs_i == 4) {
        const int *e = h_rs_err.p + (long)(nf - 1) * 4;
        f.rs_avg = (e[0] + e[1] + e[2] + e[3]) / 4;
    }
    f.out_frames += kept;
    f.total_frames += kept;
}

void FrameStage::count_rs(Fec &f, int nf, int rs_i)
{
    for (long i = 0; i < (long)nf * rs_i; i++) {
        if (h_rs_err.p[i] < 0)
            f.rs_failed++;
        else
            f.rs_corrected += h_rs_err.p[i];
    }
}

void Deframer::start(Fec &f, size_t clear_bytes)
{
    fifo_bits = 32;
    state_now = 2;
    B200_CUDA(cudaMemsetAsync(fifo.p, 0, clear_bytes, f.stream));
    DefrState &S = h_dstate.p[0];
    S.state = 2;
    S.inversion = S.good = S.bad = 0;
    S.pos = 32;
    S.frame_pay = -1;
    B200_CUDA(cudaMemcpyAsync(dstate.p, h_dstate.p, sizeof(DefrState), cudaMemcpyHostToDevice, f.stream));
}

// A new stream: the lock machines, the punctured decoder's sliding buffer, the slicer and the deframers (the first 64 bytes of each bit
// FIFO are cleared). The statistics and the adaptive windows (spec_steps, tb_overlap) carry over.
void Conv::reset(Fec &f)
{
    Decoder::reset(f);
    vit_state = invalid = nrzm_last = nosync_runs = 0;
    vit.main_next_start = -1;
    vit.enc_state = 0;
    vit.hyp = VitHyp{0, 0, 0};
    idle_st = VitIdleState{-1, 0};
    last_ber = 10.f;
    swapped = 0;
    in_buffer = 0; changing_shift = 0; is_first = got_extra = false; buf_value = 128; test_bit_len = 0; pdec_start = -1;
    if (punc) {
        bdep.zero(f.stream);   // (the reference's member array: zero-initialised by the harness; never cleared afterwards)
        vitbuf.zero(f.stream);
    }
    defr.start(f, 64);
    if (two)
        defr2.start(f, 64);
    if (simple) {
        slice_par = 0;
        f.total_chunks = 0; // the hard-decision stage knows the stream's very first chunk by this count
        slice_carry.zero(f.stream);
    }
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

void Fec::open(int F, long frames_per_push)
{
    B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    for (cudaEvent_t *e : {&ev[0], &ev[1], &evm[0], &evm[1], &evf[0], &evf[1]}) // (the destructor destroys all six)
        B200_CUDA(cudaEventCreate(e));
    softbuf.alloc((size_t)cfg.max_soft + 2L * F);
    soft_tmp.alloc(2L * F);
    frames_out.alloc((size_t)(2 * frames_per_push + 4) * cadu_bytes);
}

void Decoder::reset(Fec &f)
{
    f.soft_have = 0;
    f.out_frames = 0;
    f.last_bits0 = f.last_nbits = 0;
    f.rs_avg = 0;
    f.done_bits.clear();
    f.pulled_bits.clear();
    tail_seen = -1;
    base_off = 0;
    last_nf = 0;
}

// A push's records, timings and debug bits start empty, unless it brought no new bytes (then it changes nothing).
bool Decoder::begin(Fec &f, int F)
{
    if (f.soft_have == tail_seen)
        return false;
    last_nf = 0;
    for (float &t : t_ms)
        t = 0;
    f.last_bits0 = f.last_nbits = 0;
    f.t_frames = 0;
    if (f.soft_have < F) {
        tail_seen = f.soft_have;
        return false;
    }
    return true;
}

void Decoder::end(Fec &f)
{
    B200_CUDA(cudaEventRecord(f.ev[1], f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&f.t_vit, f.ev[0], f.ev[1]);
}

void Correlated::alloc(long positions, long frames_cap)
{
    score.alloc((size_t)positions);
    bsync.alloc((size_t)positions);
    bval.alloc((size_t)positions / 32 + 2);
    bidx.alloc((size_t)positions / 32 + 2);
    max_frames = frames_cap;
    frames.alloc((size_t)max_frames);
    walk.alloc(1);
    h_walk.alloc(1);
    h_frames.alloc((size_t)max_frames);
}

void Correlated::reset(Fec &f)
{
    Decoder::reset(f);
    lock = 0;
    cor = 0.f;
}

void Correlated::stats(b200_fec_stats *o)
{
    o->correlator_lock = lock;
    o->correlator_corr = cor;
    o->ldpc_resyncs = resyncs;
}

int Correlated::walked(cudaStream_t stream)
{
    B200_CUDA(cudaMemcpyAsync(h_walk.p, walk.p, sizeof(WalkOut), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    return h_walk.p->nf;
}

// after keep_soft_tail: `soft_have` is what the FIFO keeps
void Correlated::finish(int nf, long soft_have)
{
    for (int k = 0; k < nf; k++) {
        WalkFrame &r = h_frames.p[k];
        r.off += base_off;
        resyncs += r.pos != 0;
    }
    if (nf > 0) {
        lock = h_frames.p[nf - 1].pos == 0;
        cor = h_frames.p[nf - 1].cor;
    }
    last_nf = nf;
    base_off += h_walk.p->next;
    tail_seen = soft_have;
}

void Deframer::alloc(Fec &f, long max_new_bits, int cadu_size_, uint32_t asm_sync_, int st_synced_, int st_syncing_)
{
    cadu_size = cadu_size_;
    asm_sync = asm_sync_;
    st_synced = st_synced_;
    st_syncing = st_syncing_;
    fifo.alloc((size_t)((max_new_bits + 2L * cadu_size + 4096) / 32 + 8));
    dstate.alloc(2);
    h_dstate.alloc(1);
    max_events = defr_event_cap(32L * (long)fifo.n, cadu_size);
    devents.alloc((size_t)max_events);
    h_events.alloc((size_t)max_events);
    start(f, fifo.n * sizeof(uint32_t));
}

void FrameStage::alloc(Fec &f, long max_frames_, int rs_i, bool usecheck)
{
    max_frames = max_frames_;
    const size_t nrs = (size_t)(max_frames + 4) * std::max(1, rs_i);
    frames.alloc((size_t)max_frames);
    frames_tmp.alloc(usecheck ? (size_t)(max_frames + 4) * f.cadu_bytes : 1);
    rs_err.alloc(nrs);
    h_rs_err.alloc(nrs);
    frame_dst.alloc((size_t)max_frames + 4);
    counters.alloc(8);
    h_counters.alloc(8);
    tables.alloc(1);
    RsTables T;
    build_rs_tables(T);
    B200_CUDA(cudaMemcpyAsync(tables.p, &T, sizeof(T), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream)); // (T dies here)
    smem = (int)sizeof(RsTables) + ((f.cadu_bytes + 15) & ~15) + RS_MAX_I * 704;
    // (the limit belongs to the kernel, not to this handle: it is set for the largest CADU, 65536 bits, so that no handle lowers it
    // below what another one launches with)
    B200_CUDA(cudaFuncSetAttribute(k_frames, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(RsTables) + 8192 + RS_MAX_I * 704));
}

void Fec::reset()
{
    DeviceGuard g(cfg.device);
    B200_CUDA(cudaStreamSynchronize(stream));
    decoder->reset(*this);
}

void Deframer::compact(Fec &f)
{
    DefrState S = *h_dstate.p;
    long keep = S.frame_pay >= 0 ? S.frame_pay : S.pos - 31;
    keep = std::max<long>(0, std::min<long>(keep, fifo_bits));
    const long keep_al = keep & ~31L;
    if (keep_al > 0) {
        const long nwords = ((fifo_bits - keep_al) + 31) / 32 + 1;
        k_words_move<<<1, 1024, 0, f.stream>>>(fifo.p, fifo.p + keep_al / 32, nwords);
        f.launches++;
        S.pos -= keep_al;
        if (S.frame_pay >= 0)
            S.frame_pay -= keep_al;
        fifo_bits -= keep_al;
        *h_dstate.p = S;
        B200_CUDA(cudaMemcpyAsync(dstate.p, h_dstate.p, sizeof(DefrState), cudaMemcpyHostToDevice, f.stream));
    }
}

// Saves the machine (device state into its slot 1, host mirror) and the frame counters, for a rollback by rewind().
Deframer::Mark Deframer::mark(const Fec &f)
{
    B200_CUDA(cudaMemcpyAsync(dstate.p + 1, dstate.p, sizeof(DefrState), cudaMemcpyDeviceToDevice, f.stream));
    return Mark{h_dstate.p[0], fifo_bits, f.out_frames, f.total_frames, f.rs_corrected, f.rs_failed, state_now};
}
void Deframer::rewind(Fec &f, const Mark &m)
{
    B200_CUDA(cudaMemcpyAsync(dstate.p, dstate.p + 1, sizeof(DefrState), cudaMemcpyDeviceToDevice, f.stream));
    h_dstate.p[0] = m.h_dstate;
    fifo_bits = m.fifo_bits;
    f.out_frames = m.out_frames;
    f.total_frames = m.total_frames;
    f.rs_corrected = m.rs_corrected;
    f.rs_failed = m.rs_failed;
    state_now = m.state_now;
}

int last_raw_bit(Fec &f, const uint32_t *chunk_bits, int bit_words, long q, int nbits)
{
    uint32_t w;
    const int k = nbits - 1;
    B200_CUDA(cudaMemcpyAsync(&w, chunk_bits + q * bit_words + (k >> 5), 4, cudaMemcpyDeviceToHost, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream));
    return (w >> (31 - (k & 31))) & 1;
}

// The regions overlap only if left > used; then the copy goes through soft_tmp.
void Fec::keep_soft_tail(long used)
{
    const long left = soft_have - used;
    if (used > 0 && left > 0) {
        if (left <= used)
            B200_CUDA(cudaMemcpyAsync(softbuf.p, softbuf.p + used, left, cudaMemcpyDeviceToDevice, stream));
        else {
            B200_REQUIRE((size_t)left <= soft_tmp.n, B200_ESTATE, "internal: %ld soft bytes to keep, more than the scratch's %zu", left, soft_tmp.n);
            B200_CUDA(cudaMemcpyAsync(soft_tmp.p, softbuf.p + used, left, cudaMemcpyDeviceToDevice, stream));
            B200_CUDA(cudaMemcpyAsync(softbuf.p, soft_tmp.p, left, cudaMemcpyDeviceToDevice, stream));
        }
    }
    soft_have = left;
}

// ccsds_simple_psk_decoder: module_ccsds_simple_psk_decoder.cpp:144-296 over the nch complete cadu_size-byte chunks of the soft FIFO
void Conv::decode_simple(Fec &f, long nch)
{
    if (nch == 0)
        return;
    const int n = f.chunk;
    const bool qpsk = f.cfg.constellation == B200_QPSK;
    B200_REQUIRE(((defr.fifo_bits + nch * (long)n + 64) >> 5) + 2 < (long)defr.fifo.n, B200_ESTATE, "internal: bit FIFO too small");
    SliceCfg P;
    P.n = n;
    P.bit_words = slice_words;
    P.qpsk = qpsk;
    P.nrzm = f.cfg.nrzm;
    P.swap_iq = f.cfg.qpsk_swap_iq;
    P.swap_diff = f.cfg.qpsk_swap_diff;
    P.delay = f.cfg.oqpsk_delay;
    const long words = nch * ((n + 31) / 32);
    k_slice<<<(unsigned)std::min<long>((words + 255) / 256, 132 * 16), 256, 0, f.stream>>>(f.softbuf.p, nch, P, f.total_chunks, slice_carry.p + 2 * slice_par,
                                                                                       slice_carry.p + 2 * (slice_par ^ 1), two ? slice_bits2.p : nullptr,
                                                                                       slice_bits.p);
    slice_par ^= 1;
    f.launches++;
    const bool bpsk_nrzm = !qpsk && f.cfg.nrzm;
    // one pass over chunks [c0, c0 + m): second deframer first, then the main one (the order of one reference iteration); true when
    // both found frames
    auto run = [&](long c0, long m) {
        int nfa = 0;
        if (two) {
            k_bits_append<<<1024, 256, 0, f.stream>>>(slice_bits2.p + c0 * slice_words, m, n, slice_words, 0, 0, defr2.fifo.p, defr2.fifo_bits);
            f.launches++;
            nfa = defr2.deframe(f, fs, m * (long)n);
        }
        const int last_raw = bpsk_nrzm ? last_raw_bit(f, slice_bits.p, slice_words, c0 + m - 1, n) : 0;
        k_bits_append<<<1024, 256, 0, f.stream>>>(slice_bits.p + c0 * slice_words, m, n, slice_words, bpsk_nrzm, nrzm_last, defr.fifo.p, defr.fifo_bits);
        f.launches++;
        const int nfb = defr.deframe(f, fs, m * (long)n);
        if (bpsk_nrzm)
            nrzm_last = last_raw;
        return nfa > 0 && nfb > 0;
    };
    if (!two || nch == 1)
        run(0, nch);
    else {
        // both deframers finding frames in the same call is all but impossible for a real signal; if it happens the
        // reference's output order is per iteration, so redo this call one chunk at a time
        const Deframer::Mark m1 = defr.mark(f), m2 = defr2.mark(f);
        if (run(0, nch)) {
            f.replays++;
            defr.rewind(f, m1);
            defr2.rewind(f, m2);
            for (long c = 0; c < nch; c++)
                run(c, 1);
        }
    }
    f.total_bits += nch * (long)n;
    f.last_nbits += nch * (long)n;
}

// metop_ahrpt_decoder / ccsds_conv_concat_decoder: Viterbi (or its depunctured form) -> NRZ-M -> deframer -> RS over the nch soft
// chunks of the FIFO
void Conv::decode_conv(Fec &f, long nch)
{
    const int F = vit.geom.F;
    long c = 0;
    std::vector<OutChunk> outs;
    while (c < nch) {
        const Deframer::Mark m0 = defr.mark(f); // for the (rare) MetOp "deframer stuck in NOSYNC -> viterbi.reset()" rollback
        if (punc)
            punc_segment(f, c, nch, outs);
        else
            viterbi_segment(f, c, nch, outs);
        const long nout = (long)outs.size();
        long next_c = nch;
        if (nout > 0) {
            B200_REQUIRE(((defr.fifo_bits + nout * F + 64) >> 5) + 2 < (long)defr.fifo.n, B200_ESTATE, "internal: bit FIFO too small");
            const int last_raw = f.cfg.nrzm ? last_raw_bit(f, vit.chunk_bits.p, vit.geom.bit_words, nout - 1, F) : 0;
            k_bits_append<<<1024, 256, 0, f.stream>>>(vit.chunk_bits.p, nout, F, vit.geom.bit_words, f.cfg.nrzm, nrzm_last, defr.fifo.p, defr.fifo_bits);
            f.launches++;
            defr.deframe(f, fs, nout * (long)F);
            long redo_from = -1;
            if (metop) {
                // module_metop_ahrpt_decoder.cpp:59-72: ten consecutive decoder calls that end with the deframer in NOSYNC reset the Viterbi
                const int ne = defr.n_events;
                int ei = 0, st = 0;
                {   // state before this segment = snapshot
                    DefrState snap;
                    B200_CUDA(cudaMemcpyAsync(&snap, defr.dstate.p + 1, sizeof(DefrState), cudaMemcpyDeviceToHost, f.stream));
                    B200_CUDA(cudaStreamSynchronize(f.stream));
                    st = snap.state;
                }
                for (long k = 0; k < nout; k++) {
                    const long end = m0.fifo_bits + (k + 1) * (long)F; // exclusive
                    while (ei < ne && defr.h_events.p[ei].pos < end)
                        st = defr.h_events.p[ei++].state;
                    if (st == 2) {
                        if (++nosync_runs >= 10) {
                            nosync_runs = 0;
                            // viterbi.reset() after output chunk k. If the decoder had lost lock at exactly this chunk anyway, what
                            // follows was already decoded from the IDLE state with the same carried registers: nothing to redo.
                            if (outs[k].state_after == 0)
                                continue;
                            redo_from = k;
                            break;
                        }
                    } else
                        nosync_runs = 0;
                }
            }
            if (redo_from >= 0 && redo_from < nout - 1) {
                // roll back to just after output chunk redo_from, with the Viterbi forced to IDLE
                f.replays++;
                const OutChunk &oc = outs[redo_from];
                defr.rewind(f, m0);
                defr.deframe(f, fs, (redo_from + 1) * (long)F);
                vit_state = 0;
                vit.main_next_start = oc.next_start;
                vit.enc_state = oc.enc_tail;
                idle_st = oc.idle_st;
                invalid = oc.invalid_after;
                nosync_runs = 0;
                next_c = oc.soft_chunk + 1;
                f.total_bits += (redo_from + 1) * (long)F;
                f.last_nbits += (redo_from + 1) * (long)F;
            } else {
                if (redo_from >= 0)
                    vit_state = 0; // reset after the last chunk: nothing to redo
                if (f.cfg.nrzm)
                    nrzm_last = last_raw;
                f.total_bits += nout * (long)F;
                f.last_nbits += nout * (long)F;
            }
        }
        c = next_c;
    }
}

// rotate_soft(buffer, size, PHASE_0, true) of ccsds_conv_concat_decoder with "bpsk_90" or "iq_invert"
// (module_ccsds_conv_concat_decoder.cpp:149-150): the two bytes of every soft pair swapped, pairs counted from the stream's start
static __global__ void k_swap_pairs(int8_t *__restrict__ soft, long npairs)
{
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npairs; i += (long)gridDim.x * blockDim.x) {
        const int8_t t = soft[2 * i];
        soft[2 * i] = soft[2 * i + 1];
        soft[2 * i + 1] = t;
    }
}

void Fec::process()
{
    DeviceGuard g(cfg.device);
    decoder->process(*this);
}

void Conv::process(Fec &f)
{
    cudaStream_t stream = f.stream;
    if (f.cfg.kind == B200_FEC_CCSDS && (f.cfg.constellation == B200_BPSK_90 || f.cfg.iq_invert)) {
        // every complete pair not swapped yet (the FIFO starts on a pair boundary: chunks are even)
        const long npairs = (f.soft_have & ~1L) / 2 - swapped / 2;
        if (npairs > 0) {
            k_swap_pairs<<<(unsigned)std::min<long>((npairs + 255) / 256, 132 * 16), 256, 0, stream>>>(f.softbuf.p + swapped, npairs);
            f.launches++;
            swapped += 2 * npairs;
        }
    }
    const long nch = f.soft_have / f.chunk;
    B200_REQUIRE(nch <= max_chunks, B200_ESTATE, "internal: too many chunks");
    // (lazy, so that b200_fec_debug_bits can still read the previous push's bits until now)
    defr.compact(f);
    if (two)
        defr2.compact(f);
    f.last_bits0 = defr.fifo_bits;
    f.last_nbits = 0;
    f.t_frames = 0;
    f.t_vit_main = 0;
    f.last_main_chunks = 0;
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    if (simple)
        decode_simple(f, nch);
    else
        decode_conv(f, nch);
    f.total_chunks += nch;
    f.keep_soft_tail(nch * (long)f.chunk);
    swapped = std::max(0L, swapped - nch * (long)f.chunk);
    end(f);
    f.t_vit -= f.t_frames; // ev[0]..ev[1] spans both stages
}

long Fec::pull(uint8_t *host_out, long cap)
{
    DeviceGuard g(cfg.device);
    const long nb = out_frames * cadu_bytes;
    B200_REQUIRE(nb <= cap, B200_ESTATE, "output buffer too small: need %ld bytes", nb);
    if (nb > 0) {
        B200_CUDA(cudaMemcpyAsync(host_out, frames_out.p, nb, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
    }
    const long kb = std::min<long>((long)done_bits.size(), out_frames);
    pulled_bits.assign(done_bits.end() - kb, done_bits.end());
    done_bits.clear();
    out_frames = 0;
    return nb;
}

// The counters of the handle, and the values a decoder reports when it has no such stage (no Viterbi: BER 10, no deframer: NOSYNC)
void Fec::stats(b200_fec_stats *o)
{
    memset(o, 0, sizeof(*o));
    o->soft_in = total_soft;
    o->chunks = total_chunks;
    o->bits_out = total_bits;
    o->frames_out = total_frames;
    o->viterbi_ber = 10.f;
    o->deframer_state = 2;
    o->rs_corrected = rs_corrected;
    o->rs_failed = rs_failed;
    o->replays = replays;
    o->tb_overlap = TB_OVERLAP;
    o->kernel_launches = launches;
    o->rs_avg = rs_avg;
    decoder->stats(o);
}

void Conv::stats(b200_fec_stats *o)
{
    o->viterbi_state = vit_state;
    o->viterbi_ber = last_ber;
    o->deframer_state = defr.state_now;
    vit.stats(o);
}

void Viterbi::stats(b200_fec_stats *o) const
{
    o->replays += tb_serial_total; // start-state mis-speculations + chunks whose parallel chainback had to be redone serially
    o->start_redone = start_redone;
    o->tb_serial = tb_serial_total;
    o->spec_steps = spec_steps;
    o->tb_overlap = tb_overlap;
}

// frames in frames_out [0, out0) keep their bits; what left frames_out without a pull (b200_chain) is forgotten
void Fec::note_frame_bits(long out0, const std::vector<long> &bits)
{
    if ((long)done_bits.size() > out0)
        done_bits.erase(done_bits.begin(), done_bits.end() - out0);
    done_bits.insert(done_bits.end(), bits.begin(), bits.end());
}

long Fec::frame_bits(long *out, long cap)
{
    B200_REQUIRE(decoder->keeps_frame_bits, B200_EINVAL, "frame completion bits are kept by noaa_gac_decoder and dmsp_rtd_decoder only");
    const long n = (long)pulled_bits.size();
    B200_REQUIRE(n <= cap, B200_ESTATE, "output buffer too small: need %ld", n);
    std::copy(pulled_bits.begin(), pulled_bits.end(), out);
    return n;
}

} // namespace b200

using namespace b200;

extern "C" {
b200_fec *b200_fec_create(const b200_fec_cfg *cfg)
{
    b200_fec *h = nullptr;
    guarded([&] {
        B200_REQUIRE(cfg != nullptr, B200_EINVAL, "cfg is NULL");
        h = new b200_fec{new Fec(*cfg)};
    });
    return h;
}
void b200_fec_destroy(b200_fec *h)
{
    if (!h)
        return;
    delete h->f;
    delete h;
}
int b200_fec_push_soft(b200_fec *h, const int8_t *host_soft, long n)
{
    return guarded([&] {
        B200_REQUIRE(h && host_soft && n >= 0, B200_EINVAL, "bad argument");
        h->f->push(host_soft, n, cudaMemcpyHostToDevice);
    });
}
int b200_fec_push_soft_device(b200_fec *h, const int8_t *dev_soft, long n)
{
    return guarded([&] {
        B200_REQUIRE(h && dev_soft && n >= 0, B200_EINVAL, "bad argument");
        h->f->push(dev_soft, n, cudaMemcpyDeviceToDevice);
    });
}
int b200_fec_pull_frames(b200_fec *h, uint8_t *out, long cap, long *nbytes)
{
    return guarded([&] {
        B200_REQUIRE(h && out && nbytes, B200_EINVAL, "NULL argument");
        *nbytes = h->f->pull(out, cap);
    });
}
int b200_fec_debug_bits(b200_fec *h, uint8_t *out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        Fec &f = *h->f;
        B200_REQUIRE(f.last_nbits <= cap, B200_ESTATE, "output buffer too small: need %ld", f.last_nbits);
        B200_REQUIRE(f.last_bits0 >= 0, B200_ESTATE, "the bits of the last push are no longer in the FIFO");
        DeviceGuard g(f.cfg.device);
        const Deframer *d = f.decoder->deframer();
        const long w0 = f.last_bits0 >> 5, w1 = (f.last_bits0 + f.last_nbits + 31) >> 5;
        std::vector<uint32_t> tmp(w1 - w0 + 1);
        if (w1 > w0 && d) {
            B200_CUDA(cudaMemcpyAsync(tmp.data(), d->fifo.p + w0, (w1 - w0) * 4, cudaMemcpyDeviceToHost, f.stream));
            B200_CUDA(cudaStreamSynchronize(f.stream));
        }
        for (long i = 0; i < f.last_nbits; i++) {
            const long b = f.last_bits0 + i - (w0 << 5);
            out[i] = (tmp[b >> 5] >> (31 - (b & 31))) & 1;
        }
        *n_out = f.last_nbits;
    });
}
int b200_fec_get_stats(b200_fec *h, b200_fec_stats *out)
{
    return guarded([&] {
        B200_REQUIRE(h && out, B200_EINVAL, "NULL argument");
        h->f->stats(out);
    });
}
int b200_fec_cadu_bytes(b200_fec *h) { return h ? h->f->cadu_bytes : B200_EINVAL; }
int b200_fec_chunk_size(b200_fec *h) { return h ? h->f->chunk : B200_EINVAL; }
int b200_fec_frame_bits(b200_fec *h, long *out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        *n_out = h->f->frame_bits(out, cap);
    });
}
}
