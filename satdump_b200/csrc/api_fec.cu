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
void build_rs_tables(RsTables &T)
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

Fec::Fec(const b200_fec_cfg &in) : cfg(meteor_m2x_as_ccsds(in))
{
    const b200_fec_cfg c = cfg;
    std::unique_ptr<Framed> (*decoder)(Fec &) = nullptr; // (none: the Viterbi / simple-PSK path below)
    switch (c.kind) {
    case B200_FEC_METOP: case B200_FEC_CCSDS: case B200_FEC_SIMPLE: break;
    case B200_FEC_LDPC: decoder = ldpc_decoder; break;
    case B200_FEC_TURBO: decoder = turbo_decoder; break;
    case B200_FEC_METOP_DUMP: decoder = dump_decoder; break;
    case B200_FEC_METEOR_LRPT: decoder = meteor_decoder; break;
    case B200_FEC_NOAA_HRPT: case B200_FEC_METEOR_HRPT: case B200_FEC_DMSP_RTD: decoder = sync_walk_decoder; break;
    case B200_FEC_AQUA_DB: case B200_FEC_NOAA_GAC: decoder = bit_stage_decoder; break;
    case B200_FEC_METEOR_XBAND: decoder = xband_decoder; break;
    default: B200_REQUIRE(false, B200_EINVAL, "unknown decoder kind %d", c.kind);
    }
    B200_REQUIRE(c.max_soft >= 65536, B200_EINVAL, "max_soft must be >= 65536");
    memset(&geom, 0, sizeof(geom));
    if (decoder) {
        framed = decoder(*this);
        return;
    }
    if (c.kind != B200_FEC_METOP) {
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
    if (c.kind == B200_FEC_METOP) {
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
        spec_steps = VIT_SPEC_STEPS_34;
    } else if (c.kind == B200_FEC_SIMPLE) {
        // module_ccsds_simple_psk_decoder.cpp:19-98: one loop iteration = cadu_size soft bytes -> cadu_size bits
        B200_REQUIRE(c.constellation == B200_BPSK || c.constellation == B200_QPSK, B200_EINVAL, "CCSDS Simple PSK Decoder : invalid constellation type!");
        geom.rate34 = 0;
        geom.chunk = c.cadu_size;
        geom.F = c.cadu_size;
        nphases = 1; ph0 = ph1 = 0; nswap = 1;
        st_synced = 12;
        spec_steps = 0;
    } else {
        // module_ccsds_conv_concat_decoder.cpp:16-131
        geom.rate34 = 0;
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
        st_synced = 12;
        spec_steps = VIT_SPEC_STEPS_12;
    }
    geom.dec_stride = (geom.F + 6 + 7) & ~7;
    geom.bit_words = (geom.F + 31) / 32 + 1;
    cadu_bytes = (cfg.cadu_size + 7) / 8;
    check_device(c.device);
    DeviceGuard g(c.device);
    B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    for (auto &e : ev)
        B200_CUDA(cudaEventCreate(&e));
    for (auto &e : evm)
        B200_CUDA(cudaEventCreate(&e));
    for (auto &e : evf)
        B200_CUDA(cudaEventCreate(&e));
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
    softbuf.alloc((size_t)c.max_soft + 2 * geom.chunk);
    const bool simple = cfg.kind == B200_FEC_SIMPLE;
    dec.alloc(simple ? (size_t)(c.max_soft / 8 + geom.chunk) : (size_t)max_chunks * geom.dec_stride); // simple: only scratch for the tail move
    idle_dec.alloc(VIT_TESTLEN + 64);
    chunk_bits.alloc((size_t)max_chunks * geom.bit_words + 4);
    const long max_new_bits = max_chunks * (long)geom.F;
    fifo.alloc((size_t)((max_new_bits + 2L * cfg.cadu_size + 4096) / 32 + 8));
    start_state.alloc(max_chunks + 1);
    redo_list.alloc(2 * (size_t)max_chunks + 4); // chunk indices to decode again | chunks whose BER check follows
    h_start.resize(max_chunks + 2);
    rec.alloc(max_chunks + 1);
    tb_blocks = ((geom.F + 31) / 32 + TB_WORDS - 1) / TB_WORDS;
    tb_edges.alloc(simple ? 1 : (size_t)(max_chunks + 1) * tb_blocks);
    tb_list.alloc((size_t)max_chunks + 2); // chunks whose parallel chainback blocks disagreed at an edge (any number: low SNR makes them common)
    idle_out.alloc(1);
    idle2_out.alloc(1);
    h_idle2.alloc(1);
    B200_CUDA(cudaFuncSetAttribute(k_vit_idle2, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * VIT_IDLE_WARP_BYTES));
    dstate.alloc(2);
    devents.alloc(4096);
    if (simple) {
        chunk_bits2.alloc((size_t)max_chunks * geom.bit_words + 4);
        fifo2.alloc(fifo.n);
        dstate2.alloc(2);
        slice_carry.alloc(4);
    }
    max_frames_push = max_new_bits / cfg.cadu_size + 4;
    frames.alloc(max_frames_push);
    frames_out.alloc((size_t)(2 * max_frames_push + 4) * cadu_bytes);
    frames_tmp.alloc((size_t)(max_frames_push + 4) * cadu_bytes);
    rs_err.alloc((size_t)(max_frames_push + 4) * std::max(1, cfg.rs_i));
    frame_dst.alloc((size_t)max_frames_push + 4);
    counters.alloc(8);
    tables.alloc(1);
    h_rec.alloc(max_chunks + 1);
    h_idle.alloc(1);
    h_counters.alloc(8);
    h_dstate.alloc(2);
    h_events.alloc(4096);
    h_rs_err.alloc((size_t)(max_frames_push + 4) * std::max(1, cfg.rs_i));
    RsTables T;
    build_rs_tables(T);
    B200_CUDA(cudaMemcpyAsync(tables.p, &T, sizeof(T), cudaMemcpyHostToDevice, stream));
    rec.zero(stream);
    start_stream(fifo.n * sizeof(uint32_t));
    fr_smem = (int)sizeof(RsTables) + ((cadu_bytes + 15) & ~15) + RS_MAX_I * 704;
    B200_CUDA(cudaFuncSetAttribute(k_frames, cudaFuncAttributeMaxDynamicSharedMemorySize, fr_smem));
    B200_CUDA(cudaStreamSynchronize(stream));
}

Fec::~Fec()
{
    DeviceGuard g(cfg.device);
    if (stream)
        cudaStreamSynchronize(stream);
    framed.reset();
    for (auto &e : ev)
        cudaEventDestroy(e);
    for (auto &e : evm)
        cudaEventDestroy(e);
    for (auto &e : evf)
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

struct OutChunk { long soft_chunk; int next_start, enc_tail, invalid_after, state_after; VitIdleState idle_st; };

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
// records of the whole range come back to f.h_rec. Returns the number of chunks chained back serially.
static int decode_pass(Fec &f, const int8_t *src, long c, int nrange, long out_base, int n, const int *qlist, int nber, const int *ber_list)
{
    B200_CUDA(cudaEventRecord(f.evm[0], f.stream));
    k_vit_acs3<<<(n + WPB - 1) / WPB, 32 * WPB, 0, f.stream>>>(src, c, n, f.geom, f.hyp, f.start_state.p, f.dec.p, f.rec.p, qlist);
    B200_CUDA(cudaEventRecord(f.evm[1], f.stream));
    const long nthr = (long)n * f.tb_blocks;
    B200_CUDA(cudaMemsetAsync(f.tb_list.p, 0, sizeof(int), f.stream));
    k_vit_tb<<<(unsigned)((nthr + 127) / 128), 128, 0, f.stream>>>(n, f.tb_blocks, f.geom, f.dec.p, f.chunk_bits.p, out_base, f.rec.p, f.tb_edges.p, qlist, f.tb_overlap);
    k_vit_tb_check<<<(n + 255) / 256, 256, 0, f.stream>>>(n, f.tb_blocks, f.tb_edges.p, f.tb_list.p, nrange, qlist);
    k_vit_tb_serial<<<(n + 127) / 128, 128, 0, f.stream>>>(f.tb_list.p, nrange, f.geom, f.dec.p, f.chunk_bits.p, out_base, f.rec.p); // (threads beyond the list return at once)
    k_vit_ber<<<(nber + WPB - 1) / WPB, 32 * WPB, 0, f.stream>>>(src, c, nber, f.geom, f.hyp, f.chunk_bits.p, out_base, f.enc_state, f.rec.p, ber_list);
    f.launches += 5;
    B200_CUDA(cudaMemcpyAsync(f.h_rec.p, f.rec.p, sizeof(VitRec) * nrange, cudaMemcpyDeviceToHost, f.stream));
    int tb_redone = 0;
    B200_CUDA(cudaMemcpyAsync(&tb_redone, f.tb_list.p, sizeof(int), cudaMemcpyDeviceToHost, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream));
    f.tb_serial_total += tb_redone;
    float ms = 0;
    cudaEventElapsedTime(&ms, f.evm[0], f.evm[1]);
    f.t_vit_main += ms;
    return tb_redone;
}

// Optimistic parallel decode of n consecutive decoder windows (chunks c .. c+n-1 of `src`, f.geom.chunk bytes apart) into chunk_bits[out_base ..]:
// start-state speculation, one decode pass, and up to `max_rounds` redo rounds for chunks whose speculated start state was wrong. Leaves
// the per-chunk records in f.h_rec[0 .. n). Each round makes the first inconsistent chunk consistent (its predecessor is not redone), so
// n rounds always settle the range.
static void decode_range(Fec &f, const int8_t *src, long c, int n, long out_base, int max_rounds)
{
    B200_CUDA(cudaMemcpyAsync(f.start_state.p, &f.main_next_start, sizeof(int), cudaMemcpyHostToDevice, f.stream));
    if (n > 1) {
        k_vit_spec<<<(n - 1 + WPB - 1) / WPB, 32 * WPB, 0, f.stream>>>(src, c, n, f.geom, f.hyp, f.spec_steps, f.start_state.p);
        f.launches++;
    }
    const int tb_redone = decode_pass(f, src, c, n, out_base, n, nullptr, n, nullptr);
    f.last_main_chunks += n;
    if (n > 64) // the chainback warm-up follows the channel like the speculation window does
        adapt_window(f.tb_overlap, f.tb_clean, (double)tb_redone / (double)n, TB_OVERLAP, TB_OVERLAP_MAX);
    // Start states that were speculated wrong (k_vit_spec: common at low SNR, where 768 steps do not always pin the state): those
    // chunks alone are decoded again from the state their predecessor really left. A chunk's end state almost never depends on its
    // start state, so one round normally settles it; a round that changes a successor's start state is followed by another.
    for (int round = 0; round < max_rounds; round++) {
        f.h_redo.clear();
        for (int i = 1; i < n; i++)
            if (f.h_rec.p[i].start_used != f.h_rec.p[i - 1].next_start) {
                f.h_redo.push_back(i);
                f.h_start[i] = f.h_rec.p[i - 1].next_start;
            }
        if (round == 0 && n > 64) // wrong guesses: the survivors of the speculation window had not all merged (low SNR)
            adapt_window(f.spec_steps, f.spec_clean, (double)f.h_redo.size() / (double)n, f.geom.rate34 ? VIT_SPEC_STEPS_34 : VIT_SPEC_STEPS_12,
                         (f.geom.F / 32) * 32);
        if (f.h_redo.empty())
            break;
        const int m = (int)f.h_redo.size();
        f.replays += m;
        f.start_redone += m;
        // the BER check of a chunk reads the last test bits of its predecessor: redo it for the successors too
        f.h_redo_ber = f.h_redo;
        for (int i : f.h_redo)
            if (i + 1 < n)
                f.h_redo_ber.push_back(i + 1);
        std::sort(f.h_redo_ber.begin(), f.h_redo_ber.end());
        f.h_redo_ber.erase(std::unique(f.h_redo_ber.begin(), f.h_redo_ber.end()), f.h_redo_ber.end());
        const int mb = (int)f.h_redo_ber.size();
        for (int i : f.h_redo)
            B200_CUDA(cudaMemcpyAsync(f.start_state.p + i, &f.h_start[i], sizeof(int), cudaMemcpyHostToDevice, f.stream));
        B200_CUDA(cudaMemcpyAsync(f.redo_list.p, f.h_redo.data(), sizeof(int) * m, cudaMemcpyHostToDevice, f.stream));
        B200_CUDA(cudaMemcpyAsync(f.redo_list.p + n, f.h_redo_ber.data(), sizeof(int) * mb, cudaMemcpyHostToDevice, f.stream));
        decode_pass(f, src, c, n, out_base, m, f.redo_list.p, mb, f.redo_list.p + n);
    }
}

void viterbi_chained(Fec &f, const int8_t *src, long n, int *ber_errors)
{
    long c = 0;
    while (c < n) {
        const int m = (int)(n - c);
        decode_range(f, src, c, m, c, 6); // (what is still inconsistent after six rounds is decoded again below)
        int accepted = m;
        for (int i = 1; i < m; i++)
            if (f.h_rec.p[i].start_used != f.h_rec.p[i - 1].next_start) {
                f.replays++;
                accepted = i;
                break;
            }
        for (int i = 0; i < accepted; i++)
            ber_errors[c + i] = f.h_rec.p[i].ber_errors;
        f.main_next_start = f.h_rec.p[accepted - 1].next_start;
        f.enc_state = f.h_rec.p[accepted - 1].enc_tail;
        c += accepted;
    }
}

void rs_usecheck_compact(Fec &f, const uint8_t *in, int nf, int rs_i, uint8_t *out)
{
    k_frames_filter<<<1, 1024, 0, f.stream>>>(f.rs_err.p, nf, rs_i, f.frame_dst.p, f.counters.p + 2);
    k_frames_gather<<<std::min(nf, 132 * 16), 256, 0, f.stream>>>(in, f.frame_dst.p, nf, f.cadu_bytes, out);
    f.launches += 2;
    B200_CUDA(cudaMemcpyAsync(f.h_counters.p + 2, f.counters.p + 2, sizeof(int), cudaMemcpyDeviceToHost, f.stream));
}

// Viterbi over soft chunks [c0, nch): lock search while IDLE, optimistic parallel decode while SYNCED. Decoded chunks land in
// chunk_bits[0 .. nout). Returns per-output-chunk bookkeeping in `outs`.
static void viterbi_segment(Fec &f, long c0, long nch, std::vector<OutChunk> &outs)
{
    outs.clear();
    long c = c0, out_base = 0;
    const float kber = f.geom.rate34 ? 5.0f : 2.5f;
    while (c < nch) {
        if (f.vit_state == 0) {
            f.idle_st.enc_state = f.enc_state; // ONE chained CCEncoder serves the lock test and the SYNCED BER check (viterbi_3_4.cpp:126,157)
            {
                // parallel search first (one warp per hypothesis); it hands over to the serial kernel at the first chunk whose chained
                // 6-bit states its two-pass guess did not reproduce
                const int nh = f.nswap * f.nphases * 2;
                k_vit_idle2<<<1, 32 * nh, nh * VIT_IDLE_WARP_BYTES, f.stream>>>(f.softbuf.p, c, (int)(nch - c), f.geom, f.nswap, f.nphases, f.ph0, f.ph1,
                                                                               f.cfg.ber_thresold, f.idle_st, f.idle2_out.p);
                f.launches++;
                B200_CUDA(cudaMemcpyAsync(f.h_idle2.p, f.idle2_out.p, sizeof(VitIdle2Out), cudaMemcpyDeviceToHost, f.stream));
                B200_CUDA(cudaStreamSynchronize(f.stream));
                *f.h_idle.p = f.h_idle2.p->o;
                if (f.h_idle2.p->fallback_chunk >= 0) {
                    const long c2 = c + f.h_idle2.p->fallback_chunk;
                    k_vit_idle<<<1, 32, 0, f.stream>>>(f.softbuf.p, c2, (int)(nch - c2), f.geom, f.nswap, f.nphases, f.ph0, f.ph1, f.cfg.ber_thresold,
                                                      f.h_idle2.p->o.st, f.idle_dec.p, f.idle_out.p);
                    f.launches++;
                    B200_CUDA(cudaMemcpyAsync(f.h_idle.p, f.idle_out.p, sizeof(VitIdleOut), cudaMemcpyDeviceToHost, f.stream));
                    B200_CUDA(cudaStreamSynchronize(f.stream));
                    if (f.h_idle.p->lock_chunk >= 0)
                        f.h_idle.p->lock_chunk += (int)(c2 - c);
                }
            }
            f.idle_st = f.h_idle.p->st;
            f.enc_state = f.idle_st.enc_state;
            float bb = 10.f;
            for (int i = 0; i < 16; i++)
                bb = std::min(bb, f.h_idle.p->bers[i]);
            f.last_ber = bb;
            if (f.h_idle.p->lock_chunk < 0)
                break;
            c += f.h_idle.p->lock_chunk;
            f.vit_state = 1;
            f.hyp = VitHyp{f.h_idle.p->swap, f.h_idle.p->phase, f.h_idle.p->shift};
            f.invalid = 0;
            f.enc_state = f.idle_st.enc_state;
        }
        const int n = (int)(nch - c);
        decode_range(f, f.softbuf.p, c, n, out_base, 6); // (what is still inconsistent after six rounds is decoded again below)
        int accepted = 0;
        for (int i = 0; i < n; i++) {
            if (i > 0 && f.h_rec.p[i].start_used != f.h_rec.p[i - 1].next_start) {
                f.replays++; // still inconsistent after the redo rounds above: decode again from here with the true state
                break;
            }
            accepted = i + 1;
            const float ber = ((float)f.h_rec.p[i].ber_errors / (float)f.h_rec.p[i].ber_total) * kber;
            f.last_ber = ber;
            bool lost = false;
            if (ber > f.cfg.ber_thresold) { // viterbi_3_4.cpp:160-169
                f.invalid++;
                if (f.invalid > f.cfg.outsync_after) {
                    f.vit_state = 0;
                    lost = true;
                }
            } else
                f.invalid = 0;
            outs.push_back(OutChunk{c + i, f.h_rec.p[i].next_start, f.h_rec.p[i].enc_tail, f.invalid, f.vit_state, f.idle_st});
            if (lost)
                break;
        }
        f.main_next_start = f.h_rec.p[accepted - 1].next_start;
        f.enc_state = f.h_rec.p[accepted - 1].enc_tail;
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
static void punc_segment(Fec &f, long c0, long ncalls, std::vector<OutChunk> &outs)
{
    outs.clear();
    const int V = f.geom.chunk, size = f.geom.chunk;
    const PuncTab &P = f.ptab;
    auto made = [&](long m) { return (m / P.P) * (long)P.Q + P.cum[m % P.P]; };
    long c = c0, out_base = 0;
    while (c < ncalls) {
        if (f.vit_state == 0) {
            const VitIdleState st{f.pdec_start, f.enc_state};
            k_punc_idle<<<1, 32, 0, f.stream>>>(f.softbuf.p, c, (int)(ncalls - c), size, P, f.nswap, f.nphases, f.ph0, f.ph1, f.cfg.ber_thresold, st, f.bdep.p,
                                                f.idle_dec.p, f.punc_out.p);
            f.launches++;
            B200_CUDA(cudaMemcpyAsync(f.h_punc.p, f.punc_out.p, sizeof(PuncIdleOut), cudaMemcpyDeviceToHost, f.stream));
            B200_CUDA(cudaStreamSynchronize(f.stream));
            const PuncIdleOut &o = *f.h_punc.p;
            f.pdec_start = o.st.dec_start;
            f.enc_state = o.st.enc_state;
            f.test_bit_len = o.test_bit_len;
            f.last_ber = o.ber;
            if (o.lock_call < 0)
                break;
            c += o.lock_call;
            f.vit_state = 1;
            f.hyp = VitHyp{o.swap, o.phase, 0};
            f.invalid = 0;
            f.changing_shift = o.shift; // set_shift (depunc.h)
            f.is_first = o.shift > P.P - 1;
        }
        const int n = (int)(ncalls - c);
        // depunc_cont of calls c .. c+n-1. A symbol held back by the previous call (got_extra) already sits at vitbuf[in_buffer].
        const int held = f.got_extra ? 1 : 0;
        const int lead = (!f.got_extra && f.is_first) ? 1 : 0; // `buf` emitted in front (its stale value when nothing is held)
        f.is_first = false;
        const int a0 = f.changing_shift % P.P;
        const long nsoft = (long)n * size;
        B200_REQUIRE((size_t)(f.in_buffer + held + lead + made(a0 + nsoft) - made(a0) + 16) <= f.vitbuf.n, B200_ESTATE, "internal: depunctured stream buffer too small");
        k_punc_depunc<<<(unsigned)((nsoft + 255) / 256), 256, 0, f.stream>>>(f.softbuf.p + c * (long)size, nsoft, f.hyp, P, a0, lead, f.buf_value,
                                                                            f.vitbuf.p + f.in_buffer + held);
        f.launches++;
        // which call decodes which window, and how much of its 12-symbol tail exists by then
        f.h_tail.clear();
        f.h_wcall.clear();
        long w = 0;
        for (int j = 1; j <= n; j++) {
            const long raw = held + lead + made(a0 + (long)j * size) - made(a0);
            const long T = f.in_buffer + 2 * (raw / 2);
            while (T - w * V > V) {
                f.h_wcall.push_back(j);
                f.h_tail.push_back((int)std::min<long>(12, T - (w + 1) * V));
                w++;
            }
        }
        const int nw = (int)w;
        B200_REQUIRE(nw >= 1 && nw <= f.max_chunks, B200_ESTATE, "internal: window count %d out of range", nw);
        B200_CUDA(cudaMemcpyAsync(f.tail_real.p, f.h_tail.data(), sizeof(int) * nw, cudaMemcpyHostToDevice, f.stream));
        f.geom.tail_real = f.tail_real.p;
        f.geom.ber_bits = VIT_TESTLEN;      // cc_encoder_ber.work(output, ...) encodes TEST_BITS_LENGTH bits (viterbi_punc.cpp:124)
        f.geom.ber_syms = f.test_bit_len;   // get_ber(vit_buffer, ..., test_bit_len, 5) (:125)
        // the lock machine below accepts windows call by call and has no way back to a window decoded from a wrong start state, so the
        // redo rounds run until every window's start state is its predecessor's next start
        decode_range(f, reinterpret_cast<const int8_t *>(f.vitbuf.p), 0, nw, out_base, nw);
        // replay the lock machine call by call
        int jacc = n, wacc = nw;
        for (int j = 1, wi = 0; j <= n; j++) {
            int last = -1;
            while (wi < nw && f.h_wcall[wi] == j)
                last = wi++;
            if (last >= 0)
                f.last_ber = ((float)f.h_rec.p[last].ber_errors / (float)f.h_rec.p[last].ber_total) * 5.0f;
            if (f.last_ber > f.cfg.ber_thresold) { // viterbi_punc.cpp:133-141
                f.invalid++;
                if (f.invalid > f.cfg.outsync_after) {
                    f.vit_state = 0;
                    jacc = j;
                    wacc = wi;
                    break;
                }
            } else
                f.invalid = 0;
        }
        for (int i = 0; i < wacc; i++)
            outs.push_back(OutChunk{c + f.h_wcall[i] - 1, f.h_rec.p[i].next_start, f.h_rec.p[i].enc_tail, f.invalid, f.vit_state, f.idle_st});
        if (wacc > 0) {
            f.main_next_start = f.h_rec.p[wacc - 1].next_start;
            f.enc_state = f.h_rec.p[wacc - 1].enc_tail;
        }
        // what stays in the sliding buffer: the symbols behind the decoded windows up to the last accepted call's total, plus the one
        // that call held back (its value is DepuncXX::buf from now on)
        const long raw = held + lead + made(a0 + (long)jacc * size) - made(a0);
        const long T = f.in_buffer + 2 * (raw / 2);
        f.got_extra = raw & 1;
        f.changing_shift = (int)((a0 + (long)jacc * size) % P.P);
        const long keep0 = (long)wacc * V, keep = T - keep0 + (f.got_extra ? 1 : 0);
        B200_REQUIRE(keep >= 0 && (size_t)keep <= f.vitbuf_tmp.n, B200_ESTATE, "internal: sliding buffer leftover %ld", keep);
        if (f.got_extra) {
            unsigned char hb = 0;
            B200_CUDA(cudaMemcpyAsync(&hb, f.vitbuf.p + T, 1, cudaMemcpyDeviceToHost, f.stream));
            B200_CUDA(cudaStreamSynchronize(f.stream));
            f.buf_value = hb;
        }
        if (keep > 0 && keep0 > 0) {
            B200_CUDA(cudaMemcpyAsync(f.vitbuf_tmp.p, f.vitbuf.p + keep0, keep, cudaMemcpyDeviceToDevice, f.stream));
            B200_CUDA(cudaMemcpyAsync(f.vitbuf.p, f.vitbuf_tmp.p, keep, cudaMemcpyDeviceToDevice, f.stream));
        }
        f.in_buffer = T - keep0;
        out_base += wacc;
        c += jacc;
    }
}

void Fec::deframe_and_rs(long new_bits)
{
    const long nbits = fifo_bits + new_bits;
    B200_CUDA(cudaEventRecord(evf[0], stream));
    k_deframe<<<1, 32, 0, stream>>>(fifo.p, nbits, cfg.cadu_size, st_synced, cfg.asm_sync, dstate.p, frames.p, (int)max_frames_push,
                                   reinterpret_cast<DefrEventDev *>(devents.p), 4096, counters.p);
    launches++;
    B200_CUDA(cudaMemcpyAsync(h_counters.p, counters.p, sizeof(int) * 2, cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(h_dstate.p, dstate.p, sizeof(DefrState), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(h_events.p, devents.p, sizeof(DefrEvent) * 4096, cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    const int nf = h_counters.p[0];
    last_nf = nf;
    B200_REQUIRE(nf <= max_frames_push, B200_ESTATE, "internal: frame list overflow");
    B200_REQUIRE(h_counters.p[1] <= 4096, B200_EUNSUPPORTED, "deframer changed state more than 4096 times in one push (noise input?): push smaller batches");
    if (nf > 0) {
        B200_REQUIRE((size_t)(out_frames + nf) * cadu_bytes <= frames_out.n, B200_ESTATE, "frame output buffer full: call pull_frames");
        FrameCfg fc;
        fc.cadu_bytes = cadu_bytes;
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
        uint8_t *dst = filter ? frames_tmp.p : frames_out.p + out_frames * cadu_bytes;
        k_frames<<<std::min(nf, 132 * 8), 256, fr_smem, stream>>>(fifo.p, frames.p, nf, fc, tables.p, dst, rs_err.p);
        launches++;
        int kept = nf;
        if (filter) {
            k_frames_filter<<<1, 1024, 0, stream>>>(rs_err.p, nf, cfg.rs_i, frame_dst.p, counters.p + 2);
            k_frames_gather<<<std::min(nf, 132 * 16), 256, 0, stream>>>(frames_tmp.p, frame_dst.p, nf, cadu_bytes, frames_out.p + out_frames * cadu_bytes);
            launches += 2;
            B200_CUDA(cudaMemcpyAsync(h_counters.p + 2, counters.p + 2, sizeof(int), cudaMemcpyDeviceToHost, stream));
        }
        if (cfg.rs_i > 0)
            B200_CUDA(cudaMemcpyAsync(h_rs_err.p, rs_err.p, sizeof(int) * nf * cfg.rs_i, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        if (filter)
            kept = h_counters.p[2];
        for (long i = 0; i < (long)nf * cfg.rs_i; i++) {
            if (h_rs_err.p[i] < 0)
                rs_failed++;
            else
                rs_corrected += h_rs_err.p[i];
        }
        if (cfg.rs_i == 4) {
            const int *e = h_rs_err.p + (long)(nf - 1) * 4;
            rs_avg = (e[0] + e[1] + e[2] + e[3]) / 4;
        }
        out_frames += kept;
        total_frames += kept;
    }
    B200_CUDA(cudaEventRecord(evf[1], stream));
    B200_CUDA(cudaEventSynchronize(evf[1]));
    {
        float ms = 0;
        cudaEventElapsedTime(&ms, evf[0], evf[1]);
        t_frames += ms;
    }
    fifo_bits = nbits;
    defr_state_now = h_dstate.p->state;
}

// The state a new stream starts from: the lock machines, the punctured decoder's sliding buffer and the deframers (the FIFO starts
// with 32 zero bits = the deframer's empty shifter; the first `fifo_bytes` of each bit FIFO are cleared). The statistics and the
// adaptive windows (spec_steps, tb_overlap) carry over.
void Fec::start_stream(size_t fifo_bytes)
{
    soft_have = 0;
    swapped = 0;
    fifo_bits = 32;
    vit_state = 0; invalid = 0; main_next_start = -1; enc_state = 0; nrzm_last = 0; nosync_runs = 0;
    in_buffer = 0; changing_shift = 0; is_first = got_extra = false; buf_value = 128; test_bit_len = 0; pdec_start = -1;
    if (punc) {
        bdep.zero(stream);   // (the reference's member array: zero-initialised by the harness; never cleared afterwards)
        vitbuf.zero(stream);
    }
    hyp = VitHyp{0, 0, 0};
    idle_st = VitIdleState{-1, 0};
    last_ber = 10.f;
    defr_state_now = 2;
    rs_avg = 0;
    out_frames = 0;
    last_bits0 = last_nbits = 0;
    B200_CUDA(cudaMemsetAsync(fifo.p, 0, fifo_bytes, stream));
    h_dstate.p[0].state = 2;
    h_dstate.p[0].inversion = h_dstate.p[0].good = h_dstate.p[0].bad = 0;
    h_dstate.p[0].pos = 32;
    h_dstate.p[0].frame_pay = -1;
    B200_CUDA(cudaMemcpyAsync(dstate.p, h_dstate.p, sizeof(DefrState), cudaMemcpyHostToDevice, stream));
    if (cfg.kind == B200_FEC_SIMPLE) {
        h_dstate2 = h_dstate.p[0];
        fifo_bits2 = 32;
        defr_state2 = 2;
        slice_par = 0;
        total_chunks = 0; // the hard-decision stage knows the stream's very first chunk by this count
        B200_CUDA(cudaMemsetAsync(fifo2.p, 0, fifo_bytes, stream));
        slice_carry.zero(stream);
        B200_CUDA(cudaMemcpyAsync(dstate2.p, h_dstate.p, sizeof(DefrState), cudaMemcpyHostToDevice, stream));
    }
}

// The set-up of the decoder object that every Framed decoder shares: the stream and events, the soft FIFO of max_soft + 2F bytes, the
// scratch of keep_soft_tail and the CADU output for `frames_per_push` frames a push (0: the deframer stage sizes it, deframer_storage).
void Fec::framed_storage(int F, long frames_per_push)
{
    B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    for (cudaEvent_t *e : {&ev[0], &ev[1], &evm[0], &evm[1], &evf[0], &evf[1]}) // (the destructor destroys all six)
        B200_CUDA(cudaEventCreate(e));
    softbuf.alloc((size_t)cfg.max_soft + 2L * F);
    dec.alloc((size_t)(2 * F) / sizeof(uint2) + 16);
    if (frames_per_push > 0) {
        max_frames_push = frames_per_push;
        frames_out.alloc((size_t)(2 * frames_per_push + 4) * cadu_bytes);
    }
}

void Framed::reset(Fec &f)
{
    f.soft_have = 0;
    f.out_frames = 0;
    f.done_bits.clear();
    f.pulled_bits.clear();
    tail_seen = -1;
    base_off = 0;
    last_nf = 0;
}

// A push's records, timings and debug bits start empty, unless it brought no new bytes (then it changes nothing).
bool Framed::begin(Fec &f, int F)
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

void Framed::end(Fec &f)
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
    Framed::reset(f);
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

// The deframer and frame stage behind another decoder (ccsds_ldpc_decoder's internal_stream, aqua_db_decoder): storage for `max_new_bits`
// new bits per push, as the constructor allocates it for the convolutional decoders; cfg holds the deframer's cadu_size / asm_sync and the
// frame stage's RS settings (rs_usecheck is not built here).
void Fec::deframer_storage(long max_new_bits)
{
    fifo.alloc((size_t)((max_new_bits + 2L * cfg.cadu_size + 4096) / 32 + 8));
    dstate.alloc(2);
    devents.alloc(4096);
    max_frames_push = max_new_bits / cfg.cadu_size + 4;
    frames.alloc(max_frames_push);
    frames_out.alloc((size_t)(2 * max_frames_push + 4) * cadu_bytes);
    frames_tmp.alloc(1);
    rs_err.alloc((size_t)(max_frames_push + 4) * std::max(1, cfg.rs_i));
    frame_dst.alloc((size_t)max_frames_push + 4);
    counters.alloc(8);
    tables.alloc(1);
    h_counters.alloc(8);
    h_dstate.alloc(2);
    h_events.alloc(4096);
    h_rs_err.alloc((size_t)(max_frames_push + 4) * std::max(1, cfg.rs_i));
    RsTables T;
    build_rs_tables(T);
    B200_CUDA(cudaMemcpyAsync(tables.p, &T, sizeof(T), cudaMemcpyHostToDevice, stream));
    fr_smem = (int)sizeof(RsTables) + ((cadu_bytes + 15) & ~15) + RS_MAX_I * 704;
    B200_CUDA(cudaFuncSetAttribute(k_frames, cudaFuncAttributeMaxDynamicSharedMemorySize, fr_smem));
    start_stream(fifo.n * sizeof(uint32_t));
    B200_CUDA(cudaStreamSynchronize(stream));
}

// back to the state of a freshly created decoder (new stream), keeping all allocations
void Fec::reset()
{
    DeviceGuard g(cfg.device);
    B200_CUDA(cudaStreamSynchronize(stream));
    if (framed) {
        framed->reset(*this);
        return;
    }
    start_stream(64);
    B200_CUDA(cudaStreamSynchronize(stream));
}

void Fec::swap_unit()
{
    std::swap(fifo.p, fifo2.p);
    std::swap(fifo.n, fifo2.n);
    std::swap(dstate.p, dstate2.p);
    std::swap(fifo_bits, fifo_bits2);
    std::swap(h_dstate.p[0], h_dstate2);
    std::swap(defr_state_now, defr_state2);
}

// Compacts the bit FIFO: keeps from the open frame's payload, or the 31 bits of shifter history. `sync`: wait for the upload of the
// pinned deframer mirror when one was queued (swap_unit() overwrites the mirror next).
void Fec::compact_fifo(bool sync)
{
    DefrState S = *h_dstate.p;
    long keep = S.frame_pay >= 0 ? S.frame_pay : S.pos - 31;
    keep = std::max<long>(0, std::min<long>(keep, fifo_bits));
    const long keep_al = keep & ~31L;
    if (keep_al > 0) {
        const long nwords = ((fifo_bits - keep_al) + 31) / 32 + 1;
        k_words_move<<<1, 1024, 0, stream>>>(fifo.p, fifo.p + keep_al / 32, nwords);
        launches++;
        S.pos -= keep_al;
        if (S.frame_pay >= 0)
            S.frame_pay -= keep_al;
        fifo_bits -= keep_al;
        *h_dstate.p = S;
        B200_CUDA(cudaMemcpyAsync(dstate.p, h_dstate.p, sizeof(DefrState), cudaMemcpyHostToDevice, stream));
        if (sync)
            B200_CUDA(cudaStreamSynchronize(stream));
    }
}

// Saves the main deframer (device state into its slot 1, host mirror) and the frame counters, for a rollback by rewind().
Fec::Mark Fec::mark()
{
    B200_CUDA(cudaMemcpyAsync(dstate.p + 1, dstate.p, sizeof(DefrState), cudaMemcpyDeviceToDevice, stream));
    return Mark{h_dstate.p[0], fifo_bits, out_frames, total_frames, rs_corrected, rs_failed, defr_state_now};
}
void Fec::rewind(const Mark &m)
{
    B200_CUDA(cudaMemcpyAsync(dstate.p, dstate.p + 1, sizeof(DefrState), cudaMemcpyDeviceToDevice, stream));
    h_dstate.p[0] = m.h_dstate;
    fifo_bits = m.fifo_bits;
    out_frames = m.out_frames;
    total_frames = m.total_frames;
    rs_corrected = m.rs_corrected;
    rs_failed = m.rs_failed;
    defr_state_now = m.defr_state_now;
}

// the last of the `nbits` hard bits of chunk q of chunk_bits (NRZ-M decodes the next bit against it)
int Fec::last_raw_bit(long q, int nbits)
{
    uint32_t w;
    const int k = nbits - 1;
    B200_CUDA(cudaMemcpyAsync(&w, chunk_bits.p + q * geom.bit_words + (k >> 5), 4, cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    return (w >> (31 - (k & 31))) & 1;
}

// Keeps the undecoded tail of the soft FIFO behind the `used` bytes. The regions overlap only if left > used; chunks are large, so
// then the copy goes through the head of the decision buffer.
void Fec::keep_soft_tail(long used)
{
    const long left = soft_have - used;
    if (used > 0 && left > 0) {
        if (left <= used)
            B200_CUDA(cudaMemcpyAsync(softbuf.p, softbuf.p + used, left, cudaMemcpyDeviceToDevice, stream));
        else {
            B200_CUDA(cudaMemcpyAsync(dec.p, softbuf.p + used, left, cudaMemcpyDeviceToDevice, stream));
            B200_CUDA(cudaMemcpyAsync(softbuf.p, dec.p, left, cudaMemcpyDeviceToDevice, stream));
        }
    }
    soft_have = left;
}

// ccsds_simple_psk_decoder: module_ccsds_simple_psk_decoder.cpp:144-296 over the nch complete cadu_size-byte chunks of the soft FIFO
void Fec::decode_simple(long nch)
{
    if (nch == 0)
        return;
    const int n = geom.chunk;
    const bool qpsk = cfg.constellation == B200_QPSK, two = two_deframers();
    B200_REQUIRE(((fifo_bits + nch * (long)n + 64) >> 5) + 2 < (long)fifo.n, B200_ESTATE, "internal: bit FIFO too small");
    SliceCfg P;
    P.n = n;
    P.bit_words = geom.bit_words;
    P.qpsk = qpsk;
    P.nrzm = cfg.nrzm;
    P.swap_iq = cfg.qpsk_swap_iq;
    P.swap_diff = cfg.qpsk_swap_diff;
    P.delay = cfg.oqpsk_delay;
    const long words = nch * ((n + 31) / 32);
    k_slice<<<(unsigned)std::min<long>((words + 255) / 256, 132 * 16), 256, 0, stream>>>(softbuf.p, nch, P, total_chunks, slice_carry.p + 2 * slice_par,
                                                                                     slice_carry.p + 2 * (slice_par ^ 1), two ? chunk_bits2.p : nullptr,
                                                                                     chunk_bits.p);
    slice_par ^= 1;
    launches++;
    const bool bpsk_nrzm = !qpsk && cfg.nrzm;
    // one pass over chunks [c0, c0 + m): second deframer first, then the main one (the order of one reference iteration)
    auto run = [&](long c0, long m) {
        int nfa = 0;
        if (two) {
            swap_unit();
            k_bits_append<<<1024, 256, 0, stream>>>(chunk_bits2.p + c0 * geom.bit_words, m, n, geom.bit_words, 0, 0, fifo.p, fifo_bits);
            launches++;
            deframe_and_rs(m * (long)n);
            nfa = last_nf;
            swap_unit();
        }
        const int last_raw = bpsk_nrzm ? last_raw_bit(c0 + m - 1, n) : 0;
        k_bits_append<<<1024, 256, 0, stream>>>(chunk_bits.p + c0 * geom.bit_words, m, n, geom.bit_words, bpsk_nrzm, nrzm_last, fifo.p, fifo_bits);
        launches++;
        deframe_and_rs(m * (long)n);
        if (bpsk_nrzm)
            nrzm_last = last_raw;
        return std::make_pair(nfa, last_nf);
    };
    if (!two || nch == 1)
        run(0, nch);
    else {
        // both deframers finding frames in the same call is all but impossible for a real signal; if it happens the
        // reference's output order is per iteration, so redo this call one chunk at a time
        const Mark m0 = mark();
        B200_CUDA(cudaMemcpyAsync(dstate2.p + 1, dstate2.p, sizeof(DefrState), cudaMemcpyDeviceToDevice, stream));
        const DefrState h1 = h_dstate2;
        const long fb1 = fifo_bits2;
        const int ds1 = defr_state2;
        const auto r = run(0, nch);
        if (r.first > 0 && r.second > 0) {
            replays++;
            rewind(m0);
            B200_CUDA(cudaMemcpyAsync(dstate2.p, dstate2.p + 1, sizeof(DefrState), cudaMemcpyDeviceToDevice, stream));
            h_dstate2 = h1;
            fifo_bits2 = fb1;
            defr_state2 = ds1;
            for (long c = 0; c < nch; c++)
                run(c, 1);
        }
    }
    total_bits += nch * (long)n;
    last_nbits += nch * (long)n;
}

// metop_ahrpt_decoder / ccsds_conv_concat_decoder: Viterbi (or its depunctured form) -> NRZ-M -> deframer -> RS over the nch soft
// chunks of the FIFO
void Fec::decode_conv(long nch)
{
    long c = 0;
    std::vector<OutChunk> outs;
    while (c < nch) {
        const Mark m0 = mark(); // for the (rare) MetOp "deframer stuck in NOSYNC -> viterbi.reset()" rollback
        if (punc)
            punc_segment(*this, c, nch, outs);
        else
            viterbi_segment(*this, c, nch, outs);
        const long nout = (long)outs.size();
        long next_c = nch;
        if (nout > 0) {
            B200_REQUIRE(((fifo_bits + nout * geom.F + 64) >> 5) + 2 < (long)fifo.n, B200_ESTATE, "internal: bit FIFO too small");
            const int last_raw = cfg.nrzm ? last_raw_bit(nout - 1, geom.F) : 0;
            k_bits_append<<<1024, 256, 0, stream>>>(chunk_bits.p, nout, geom.F, geom.bit_words, cfg.nrzm, nrzm_last, fifo.p, fifo_bits);
            launches++;
            deframe_and_rs(nout * (long)geom.F);
            long redo_from = -1;
            if (cfg.kind == B200_FEC_METOP) {
                // module_metop_ahrpt_decoder.cpp:59-72: ten consecutive decoder calls that end with the deframer in NOSYNC reset the Viterbi
                const int ne = h_counters.p[1];
                int ei = 0, st = 0;
                {   // state before this segment = snapshot
                    DefrState snap;
                    B200_CUDA(cudaMemcpyAsync(&snap, dstate.p + 1, sizeof(DefrState), cudaMemcpyDeviceToHost, stream));
                    B200_CUDA(cudaStreamSynchronize(stream));
                    st = snap.state;
                }
                for (long k = 0; k < nout; k++) {
                    const long end = m0.fifo_bits + (k + 1) * (long)geom.F; // exclusive
                    while (ei < ne && h_events.p[ei].pos < end)
                        st = h_events.p[ei++].state;
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
                replays++;
                const OutChunk &oc = outs[redo_from];
                rewind(m0);
                deframe_and_rs((redo_from + 1) * (long)geom.F);
                vit_state = 0;
                main_next_start = oc.next_start;
                enc_state = oc.enc_tail;
                idle_st = oc.idle_st;
                invalid = oc.invalid_after;
                nosync_runs = 0;
                next_c = oc.soft_chunk + 1;
                total_bits += (redo_from + 1) * (long)geom.F;
                last_nbits += (redo_from + 1) * (long)geom.F;
            } else {
                if (redo_from >= 0)
                    vit_state = 0; // reset after the last chunk: nothing to redo
                if (cfg.nrzm)
                    nrzm_last = last_raw;
                total_bits += nout * (long)geom.F;
                last_nbits += nout * (long)geom.F;
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
    if (framed) {
        framed->process(*this);
        return;
    }
    if (cfg.kind == B200_FEC_CCSDS && (cfg.constellation == B200_BPSK_90 || cfg.iq_invert)) {
        // every complete pair not swapped yet (the FIFO starts on a pair boundary: chunks are even)
        const long npairs = (soft_have & ~1L) / 2 - swapped / 2;
        if (npairs > 0) {
            k_swap_pairs<<<(unsigned)std::min<long>((npairs + 255) / 256, 132 * 16), 256, 0, stream>>>(softbuf.p + swapped, npairs);
            launches++;
            swapped += 2 * npairs;
        }
    }
    const long nch = soft_have / geom.chunk;
    B200_REQUIRE(nch <= max_chunks, B200_ESTATE, "internal: too many chunks");
    // (lazy, so that b200_fec_debug_bits can still read the previous push's bits until now)
    const bool simple = cfg.kind == B200_FEC_SIMPLE;
    compact_fifo(simple);
    if (two_deframers()) {
        swap_unit();
        compact_fifo(true);
        swap_unit();
    }
    last_bits0 = fifo_bits;
    last_nbits = 0;
    t_frames = 0;
    t_vit_main = 0;
    last_main_chunks = 0;
    B200_CUDA(cudaEventRecord(ev[0], stream));
    if (simple)
        decode_simple(nch);
    else
        decode_conv(nch);
    total_chunks += nch;
    keep_soft_tail(nch * (long)geom.chunk);
    swapped = std::max(0L, swapped - nch * (long)geom.chunk);
    B200_CUDA(cudaEventRecord(ev[1], stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&t_vit, ev[0], ev[1]);
    t_vit -= t_frames; // ev[0]..ev[1] spans both stages
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

void Fec::stats(b200_fec_stats *o)
{
    memset(o, 0, sizeof(*o));
    o->soft_in = total_soft;
    o->chunks = total_chunks;
    o->bits_out = total_bits;
    o->frames_out = total_frames;
    o->viterbi_state = vit_state;
    o->viterbi_ber = last_ber;
    o->deframer_state = defr_state_now;
    o->rs_corrected = rs_corrected;
    o->rs_failed = rs_failed;
    o->replays = replays + tb_serial_total; // start-state mis-speculations + chunks whose parallel chainback had to be redone serially
    o->start_redone = start_redone;
    o->tb_serial = tb_serial_total;
    o->spec_steps = spec_steps;
    o->tb_overlap = tb_overlap;
    o->kernel_launches = launches;
    o->rs_avg = rs_avg;
    if (framed)
        framed->stats(o);
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
        const long w0 = f.last_bits0 >> 5, w1 = (f.last_bits0 + f.last_nbits + 31) >> 5;
        std::vector<uint32_t> tmp(w1 - w0 + 1);
        if (w1 > w0) {
            B200_CUDA(cudaMemcpyAsync(tmp.data(), f.fifo.p + w0, (w1 - w0) * 4, cudaMemcpyDeviceToHost, f.stream));
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
int b200_fec_chunk_size(b200_fec *h) { return h ? h->f->geom.chunk : B200_EINVAL; }
int b200_fec_frame_bits(b200_fec *h, long *out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        *n_out = h->f->frame_bits(out, cap);
    });
}
}
