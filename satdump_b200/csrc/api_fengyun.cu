// Host driver of the two FengYun-3 decoders over the soft FIFO of Fec, in the modules' 16384-byte reads counted from the stream's start:
//   fengyun_ahrpt_decoder (B200_FEC_FENGYUN_AHRPT)  FengyunAHRPTDecoderModule::process
//                                                    (plugins/fengyun3_support/fengyun3/module_fengyun_ahrpt_decoder.cpp:42-136)
//   fengyun_mpt_decoder (B200_FEC_FENGYUN_MPT)      FengyunMPTDecoderModule::process
//                                                    (plugins/fengyun3_support/fengyun3/module_fengyun_mpt_decoder.cpp:42-135)
// Every read: k_fy_split -> two Viterbis (Viterbi3_4 fymode / Viterbi1_2) -> FengyunDiff::work2 (k_fy_diff) -> when both Viterbis
// decoded, the deframer and the frame stage of the convolutional decoders. What differs between the two modules is data (FyKind).
//
// The module's search machines change only at read boundaries:
//   * shift: after a read that leaves a Viterbi in NOSYNC (AHRPT: either one; MPT: viterbi1 only, as the module's test names viterbi1
//     twice), viterbiNoSyncRun++ (never reset); from 10 on, every such read toggles shift. It decides how the next reads are split,
//     so the driver splits a run of reads with the current shift, decodes both branches,
//     walks the reads on the host and, at the first toggle, rolls both Viterbis back to the end of that read and splits the rest again.
//     While both Viterbis are SYNCED nothing toggles, so a locked push is split and decoded as one run. While one of them is in NOSYNC
//     the driver steps read by read (the lock search reports the BERs of every read).
//   * invert_branches: after 10 reads in a row that leave the deframer in NOSYNC (counted on reads where both Viterbis decoded) the
//     branches swap in front of the differential decoder. The deframer runs speculatively over all of a run's reads, and at a swap it
//     rewinds to the run's start, walks up to that read again and continues with the swapped branches (the MetOp rollback).
#include "fengyun.cuh"
#include "fec_host.h"
#include <algorithm>

namespace b200
{

// What distinguishes fengyun_mpt_decoder from fengyun_ahrpt_decoder
struct FyKind
{
    const char *name;
    int rate34;                       // the Viterbi: 1 Viterbi3_4(fymode), 0 Viterbi1_2 (VitGeom::rate34; its BER scale follows)
    int F;                            // bits one Viterbi call returns per branch and read
    int spec_steps;                   // k_vit_spec's initial window
    int nphases, ph0, ph1;            // the lock search's phases (one I/Q-swap hypothesis, both shifts)
    int idle_mode;                    // the lock search's VIT_IDLE_*: FY, FengYun's depuncture, VitHyp{shift, phase, shift}; else
                                      // VitHyp{swap, phase, shift}
    int st_syncing, st_synced;        // the deframer's STATE_SYNCING / STATE_SYNCED
    bool v2_toggles;                  // a read leaving viterbi2 in NOSYNC counts towards the shift toggle
    bool invert_q;                    // the module has invert_second_viterbi (else Q is always complemented and a nonzero one is refused)
    void (*split)(const int8_t *, long, int, int, int8_t *, int8_t *);
    void (*diff)(const uint32_t *, const uint32_t *, int, const int *, int, int, int, int, uint32_t *, long);
};
static const FyKind FY_AHRPT{"fengyun_ahrpt_decoder", 1, FY_BITS, VIT_SPEC_STEPS_34, 1, 0, 0, VIT_IDLE_FY, 8, 16, true, true, k_fy_split<false>,
                             k_fy_diff<FY_BITS>};
static const FyKind FY_MPT{"fengyun_mpt_decoder", 0, FY_MPT_BITS, VIT_SPEC_STEPS_12, 2, 0, 1, VIT_IDLE_R12_EXACT, 6, 12, false, false,
                           k_fy_split<true>, k_fy_diff<FY_MPT_BITS>};

// One Viterbi3_4(ber, outsync, 8192, fymode = true) (viterbi_3_4.cpp:106-173) or Viterbi1_2(ber, outsync, 8192, {PHASE_0, PHASE_90})
// (viterbi_1_2.cpp:36-116) and its lock machine, decoding one branch of the reads
struct FyVit
{
    struct State
    {
        int vit_state = 0, invalid = 0;
        VitIdleState idle_st{-1, 0};
        unsigned idle_head = 0;       // (Viterbi1_2) the first bits the last lock trial decoded
        VitHyp hyp{0, 0, 0};
        int main_next_start = -1, enc_state = 0;
        float ber = 10.f, search_ber = 10.f; // ber(): SYNCED the last BER check, else the least BER of the last lock search
    };
    struct ReadOut { int bits; State after; };
    Viterbi vit;
    DevBuf<int8_t> soft;              // the branch of the reads being decoded, FY_BRANCH bytes each (k_fy_split)
    State s;
    std::vector<ReadOut> outs;        // per read of the run: what work() returned and the machine after it

    State now() const
    {
        State t = s;
        t.hyp = vit.hyp;
        t.main_next_start = vit.main_next_start;
        t.enc_state = vit.enc_state;
        return t;
    }
    void restore(const State &t)
    {
        s = t;
        vit.hyp = t.hyp;
        vit.main_next_start = t.main_next_start;
        vit.enc_state = t.enc_state;
    }
    // SYNCED: reads j .. j + m - 1 decoded as one range; appends the reads accepted (at least one), up to and with a read that loses the lock
    void decode(Fec &f, long j, int m)
    {
        vit.decode_range(f, soft.p, j, m, j, 6); // (what is still inconsistent after six rounds is decoded again by the next call)
        const VitRec *rec = vit.h_rec.p;
        for (int i = 0; i < m; i++) {
            if (i > 0 && rec[i].start_used != rec[i - 1].next_start) {
                f.replays++;
                break;
            }
            const float ber = ((float)rec[i].ber_errors / (float)rec[i].ber_total) * (vit.geom.rate34 ? 5.0f : 2.5f);
            bool lost = false;
            if (ber > f.cfg.ber_thresold) { // viterbi_3_4.cpp:160-169, viterbi_1_2.cpp:99-109
                if (++s.invalid > f.cfg.outsync_after) {
                    s.vit_state = 0;
                    lost = true;
                }
            } else
                s.invalid = 0;
            s.ber = lost ? s.search_ber : ber;
            vit.main_next_start = rec[i].next_start;
            vit.enc_state = rec[i].enc_tail;
            outs.push_back(ReadOut{vit.geom.F, now()});
            if (lost)
                break;
        }
    }
    // one read: the lock search when in NOSYNC (the kind's phases, both shifts), and the read's decode when it locks or was SYNCED
    void step(Fec &f, long j, const FyKind &kind)
    {
        if (s.vit_state == 0) {
            s.idle_st.enc_state = vit.enc_state; // ONE chained CCEncoder serves the lock test and the SYNCED BER check
            const VitIdleOut &o = vit.lock_search(f, soft.p, j, 1, 1, kind.nphases, kind.ph0, kind.ph1, s.idle_st, kind.idle_mode, s.idle_head);
            s.idle_st = o.st;
            s.idle_head = o.head;
            vit.enc_state = o.st.enc_state;
            float bb = 10.f;
            for (int i = 0; i < 16; i++)
                bb = std::min(bb, o.bers[i]);
            s.search_ber = s.ber = bb;
            if (o.lock_chunk < 0) {
                outs.push_back(ReadOut{0, now()});
                return;
            }
            s.vit_state = 1;
            s.invalid = 0;
            // (AHRPT, k_fy_split's storage: FengYun's depuncture of shift s is the MetOp one with swap s)
            vit.hyp = VitHyp{kind.idle_mode == VIT_IDLE_FY ? o.shift : o.swap, o.phase, o.shift};
        }
        decode(f, j, 1);
    }
    void reset()
    {
        restore(State{});
    }
};

struct Fengyun : Decoder
{
    const FyKind &kind;
    FyVit v[2];                       // viterbi1 (I), viterbi2 (Q)
    Deframer defr;
    FrameStage fs;
    DevBuf<int> dreads;
    std::vector<int> act;             // reads of the run on which both Viterbis decoded
    std::vector<int> act_state, act_invert; // the deframer state and invert_branches after each of them
    int shift = 0, invert = 0, nosync_runs = 0, vit_nosync_runs = 0;
    int xin = 0, yin = 0;             // FengyunDiff's Xin >> 1 and Yin: the last pair it took
    long reads_done = 0;
    std::vector<b200_fengyun_read> recs; // the last push's

    Fengyun(Fec &f, const FyKind &k);
    void process(Fec &f) override;
    void reset(Fec &f) override;
    void stats(b200_fec_stats *o) override;
    const Deframer *deframer() const override { return &defr; }
    int run_reads(Fec &f, long r, int n);
    void frames(Fec &f, int e);
};

Fengyun::Fengyun(Fec &f, const FyKind &k) : kind(k)
{
    b200_fec_cfg &cfg = f.cfg;
    B200_REQUIRE(cfg.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for %s", kind.name);
    B200_REQUIRE(kind.invert_q || cfg.invert_second_viterbi == 0, B200_EINVAL,
                 "%s has no invert_second_viterbi: its Q branch is always complemented", kind.name);
    // BPSK_CCSDS_Deframer (8192 bits), derand_ccsds(&cadu[4], 1020), decode_interlaved(&cadu[4], true, 4): RS223 I=4 dual basis
    cfg.cadu_size = 8192;
    cfg.rs_i = 4;
    cfg.rs_dualbasis = 1;
    cfg.rs_type = 0;
    cfg.rs_fill_bytes = -1;
    cfg.rs_usecheck = 0;
    cfg.derandomize = 1;
    cfg.derand_after_rs = 0;
    cfg.derand_start = 4;
    cfg.nrzm = 0;
    cfg.asm_sync = 0x1ACFFC1D;
    f.chunk = FY_READ;
    f.cadu_bytes = 1024;
    check_device(cfg.device);
    DeviceGuard g(cfg.device);
    const long max_reads = cfg.max_soft / FY_READ + 2;
    const long max_new_bits = max_reads * 2L * kind.F;
    const long max_frames = Deframer::frames_cap(max_new_bits, cfg.cadu_size);
    f.open(FY_READ, max_frames);
    VitGeom geom{};
    geom.rate34 = kind.rate34;
    geom.chunk = FY_BRANCH;
    geom.F = kind.F;
    for (FyVit &fv : v) {
        fv.vit.spec_steps = kind.spec_steps;
        fv.vit.alloc(f, geom, max_reads);
        fv.vit.alloc_lock_search();
        fv.soft.alloc((size_t)max_reads * FY_BRANCH);
        fv.outs.reserve(max_reads);
    }
    dreads.alloc(max_reads);
    defr.alloc(f, max_new_bits, cfg.cadu_size, cfg.asm_sync, kind.st_synced, kind.st_syncing); // AHRPT module :45-46; MPT the defaults
    fs.alloc(f, max_frames, cfg.rs_i, false);
    reset(f);
}

std::unique_ptr<Decoder> fengyun_decoder(Fec &f)
{
    return std::make_unique<Fengyun>(f, f.cfg.kind == B200_FEC_FENGYUN_MPT ? FY_MPT : FY_AHRPT);
}

void Fengyun::reset(Fec &f)
{
    Decoder::reset(f);
    shift = invert = nosync_runs = vit_nosync_runs = 0;
    xin = yin = 0;
    reads_done = 0;
    recs.clear();
    for (FyVit &fv : v)
        fv.reset();
    defr.start(f, 64);
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

// Reads r .. r + n - 1 of the FIFO split with the current shift and decoded up to and with the first read that toggles shift (or all n):
// their records, bits and frames. Returns the number of reads done.
int Fengyun::run_reads(Fec &f, long r, int n)
{
    const long total = (long)n * FY_BRANCH;
    kind.split<<<(unsigned)std::min<long>((total + 255) / 256, 132 * 16), 256, 0, f.stream>>>(f.softbuf.p + r * FY_READ, n, shift,
                                                                                              f.cfg.invert_second_viterbi, v[0].soft.p, v[1].soft.p);
    f.launches++;
    for (FyVit &fv : v)
        fv.outs.clear();
    const size_t rec0 = recs.size();
    int j = 0;
    bool toggled = false;
    while (j < n && !toggled) {
        if (v[0].s.vit_state && v[1].s.vit_state) {
            v[0].decode(f, j, n - j);
            v[1].decode(f, j, n - j);
        } else {
            v[0].step(f, j, kind);
            v[1].step(f, j, kind);
        }
        int e = (int)std::min(v[0].outs.size(), v[1].outs.size());
        for (int k = j; k < e; k++) { // AHRPT module :75-86, MPT module :81-92
            const FyVit::State &a = v[0].outs[k].after, &b = v[1].outs[k].after;
            if ((a.vit_state == 0 || (kind.v2_toggles && b.vit_state == 0)) && ++vit_nosync_runs >= 10) {
                shift ^= 1;
                toggled = true;
                e = k + 1;
            }
            b200_fengyun_read R{};
            R.read = reads_done + r + k;
            R.shift = shift;
            R.v1 = v[0].outs[k].bits;
            R.v2 = v[1].outs[k].bits;
            R.state1 = a.vit_state;
            R.state2 = b.vit_state;
            R.ber1 = a.ber;
            R.ber2 = b.ber;
            recs.push_back(R);
            if (toggled)
                break;
        }
        for (FyVit &fv : v)
            if ((int)fv.outs.size() > e) { // decoded past the other one's lock loss or past a toggle: back to the end of read e - 1
                fv.restore(fv.outs[e - 1].after);
                fv.outs.resize(e);
            }
        j = e;
    }
    // the deframer state and invert_branches after every read of the run (they change only on reads where both Viterbis decoded)
    int st_run = defr.state_now, inv_run = invert;
    frames(f, j);
    size_t ai = 0;
    for (int k = 0; k < j; k++) {
        b200_fengyun_read &R = recs[rec0 + k];
        if (ai < act.size() && act[ai] == k) {
            st_run = act_state[ai];
            inv_run = act_invert[ai];
            ai++;
        }
        R.deframer_state = st_run;
        R.invert_branches = inv_run;
    }
    return j;
}

// FengyunDiff::work2 and the deframer on the reads 0 .. e - 1 of the run where both Viterbis decoded (AHRPT module :89-126, MPT :94-131)
void Fengyun::frames(Fec &f, int e)
{
    act.clear();
    act_state.clear();
    act_invert.clear();
    for (int k = 0; k < e; k++)
        if (v[0].outs[k].bits > 0 && v[1].outs[k].bits > 0)
            act.push_back(k);
    const int bw = v[0].vit.geom.bit_words;
    const long rb = 2L * kind.F; // deframer bits per read
    size_t k = 0;
    while (k < act.size()) {
        const int na = (int)(act.size() - k);
        B200_REQUIRE(((defr.fifo_bits + na * rb + 64) >> 5) + 2 < (long)defr.fifo.n, B200_ESTATE, "internal: bit FIFO too small");
        const Deframer::Mark m0 = defr.mark(f);
        const int rs_avg0 = f.rs_avg;
        B200_CUDA(cudaMemcpyAsync(dreads.p, act.data() + k, sizeof(int) * na, cudaMemcpyHostToDevice, f.stream));
        const long words = (na * rb + 64) / 32;
        kind.diff<<<(unsigned)std::min<long>((words + 255) / 256, 132 * 16), 256, 0, f.stream>>>(v[0].vit.chunk_bits.p, v[1].vit.chunk_bits.p, bw,
                                                                                               dreads.p, na, invert, xin, yin, defr.fifo.p,
                                                                                               defr.fifo_bits);
        f.launches++;
        defr.deframe(f, fs, na * rb);
        // the deframer state after each read, from the walk's state changes; NOSYNC ten reads in a row swaps the branches
        int ei = 0, st = m0.state_now, flip = -1;
        for (int a = 0; a < na; a++) {
            const long end = m0.fifo_bits + (a + 1) * rb;
            while (ei < defr.n_events && defr.h_events.p[ei].pos < end)
                st = defr.h_events.p[ei++].state;
            act_state.push_back(st);
            if (st == 2) {
                if (++nosync_runs >= 10) {
                    nosync_runs = 0;
                    flip = a;
                }
            } else
                nosync_runs = 0;
            act_invert.push_back(flip == a ? invert ^ 1 : invert);
            if (flip >= 0)
                break;
        }
        const int done = flip >= 0 ? flip + 1 : na;
        if (done < na) { // the reads behind the swap were differentially decoded with the old branch order: walk up to the swap again
            f.replays++;
            defr.rewind(f, m0);
            f.rs_avg = rs_avg0;
            defr.deframe(f, fs, done * rb);
        }
        const int q = act[k + done - 1];
        const int b0 = last_raw_bit(f, v[0].vit.chunk_bits.p, bw, q, kind.F), b1 = last_raw_bit(f, v[1].vit.chunk_bits.p, bw, q, kind.F);
        xin = invert ? b0 : b1; // in1 = viterbi2's bits unless the branches are swapped
        yin = invert ? b1 : b0;
        if (flip >= 0)
            invert ^= 1;
        f.total_bits += done * rb;
        f.last_nbits += done * rb;
        k += done;
    }
}

void Fengyun::process(Fec &f)
{
    const long seen = tail_seen;
    if (!begin(f, FY_READ)) {
        if (f.soft_have != seen) // new bytes, but no whole read: no records
            recs.clear();
        return;
    }
    B200_CUDA(cudaEventRecord(f.ev[0], f.stream));
    // (lazy, so that b200_fec_debug_bits can still read the previous push's bits until now)
    defr.compact(f);
    f.last_bits0 = defr.fifo_bits;
    f.last_nbits = 0;
    f.t_vit_main = 0;
    f.last_main_chunks = 0;
    recs.clear();
    const long nr = f.soft_have / FY_READ;
    for (long r = 0; r < nr;)
        r += run_reads(f, r, (int)(nr - r));
    reads_done += nr;
    f.total_chunks += nr;
    f.keep_soft_tail(nr * FY_READ);
    tail_seen = f.soft_have;
    last_nf = (long)recs.size();
    end(f);
    f.t_vit -= f.t_frames;
}

void Fengyun::stats(b200_fec_stats *o)
{
    o->viterbi_state = v[0].s.vit_state;
    o->viterbi_ber = v[0].s.ber;
    o->viterbi2_state = v[1].s.vit_state;
    o->viterbi2_ber = v[1].s.ber;
    o->deframer_state = defr.state_now;
    v[0].vit.stats(o);
    const long sr = o->start_redone, ts = o->tb_serial;
    v[1].vit.stats(o);
    o->start_redone += sr;
    o->tb_serial += ts;
}

} // namespace b200

using namespace b200;

extern "C" int b200_fec_debug_fengyun_reads(b200_fec *h, b200_fengyun_read *out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        const Fengyun &d = h->f->decoder_as<Fengyun>("not a fengyun_ahrpt_decoder or fengyun_mpt_decoder");
        const long n = (long)d.recs.size();
        B200_REQUIRE(n <= cap, B200_ESTATE, "output buffer too small: need %ld", n);
        std::copy(d.recs.begin(), d.recs.end(), out);
        *n_out = n;
    });
}
