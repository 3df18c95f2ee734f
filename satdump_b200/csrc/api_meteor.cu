// Host driver of meteor_lrpt_decoder with m2x_mode false (B200_FEC_METEOR_LRPT) inside the decoder object: METEORLRPTDecoderModule::process
// (plugins/meteor_support/meteor/module_meteor_lrpt_decoder.cpp:198-262) over the soft FIFO of Fec. (m2x_mode is ccsds_conv_concat_decoder's
// path: api_fec.cu.)
#include "meteor.cuh"
#include "fec_host.h"
#include <algorithm>

namespace b200
{

struct Meteor : Correlated
{
    MeteorSync sw{};
    DevBuf<uint32_t> hw;
    DevBuf<int8_t> vsoft;       // the walked frames after rotate_soft: the Viterbi decoder's chunks
    PinnedBuf<int> h_ber;       // Viterbi27's BER errors of every frame of the last push
    int nrzm = 0;

    explicit Meteor(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
    long records(const Fec &f, b200_meteor_frame *out, long cap) const; // of the last push
};

namespace
{
// correlator.cpp:3-42
uint64_t rotate_64(uint64_t word, int p)
{
    const uint64_t i = word & 0xaaaaaaaaaaaaaaaaull, q = word & 0x5555555555555555ull;
    switch (p) {
    case 1: word = ((i ^ 0xaaaaaaaaaaaaaaaaull) >> 1) | (q << 1); break;
    case 2: word = word ^ ~0ull; break;
    case 3: word = (i >> 1) | ((q ^ 0x5555555555555555ull) << 1); break;
    default: break;
    }
    return ((word & 0x5555555555555555ull) << 1) | ((word & 0xaaaaaaaaaaaaaaaaull) >> 1);
}
uint64_t swap_iq(uint64_t w) { return ((w & 0xaaaaaaaaaaaaaaaaull) >> 1) | ((w & 0x5555555555555555ull) << 1); }

// Viterbi27(8192) (common/codings/viterbi/viterbi27.cpp): frame size, and the BER test re-encodes 512 bits and compares 1024 symbols
void viterbi27_geometry(VitGeom &g)
{
    g.rate34 = 0;
    g.raw = 0;
    g.chunk = METEOR_F;
    g.F = METEOR_BITS;
    g.ber_bits = 512;
    g.ber_syms = 1024;
    g.tail_real = nullptr;
    g.dec_stride = (g.F + 6 + 7) & ~7;
    g.bit_words = (g.F + 31) / 32 + 1;
}
} // namespace

Meteor::Meteor(Fec &f)
{
    B200_REQUIRE(f.cfg.max_soft <= (1L << 28), B200_EINVAL, "max_soft must be <= 2^28 for the METEOR LRPT decoder");
    nrzm = f.cfg.diff_decode != 0;
    viterbi27_geometry(f.geom);
    f.cadu_bytes = METEOR_CADU;
    f.cfg.cadu_size = METEOR_CADU * 8;
    f.cfg.constellation = B200_QPSK;
    f.cfg.rs_i = METEOR_RS_I;
    f.spec_steps = VIT_SPEC_STEPS_12;
    f.tb_blocks = ((f.geom.F + 31) / 32 + TB_WORDS - 1) / TB_WORDS;
    f.last_ber = 0.f; // (Viterbi27's d_ber before the first frame)
    const uint64_t word = nrzm ? 0xfc4ef4fd0cc2df89ull : 0xfca2b63db00d9794ull;
    for (int p = 0; p < 4; p++) {
        sw.w[p] = rotate_64(word, p);
        sw.w[4 + p] = rotate_64(swap_iq(word) ^ ~0ull, p);
    }
    check_device(f.cfg.device);
    DeviceGuard g(f.cfg.device);
    const long fifo = f.cfg.max_soft + 2L * METEOR_F;
    alloc(fifo / 2, fifo / METEOR_F + 2); // scores at the even positions
    f.framed_storage(METEOR_F, max_frames);
    // decisions of every frame of a push; (the head also serves keep_soft_tail as scratch, after the decoder has read it)
    f.dec.alloc(std::max<size_t>((size_t)max_frames * f.geom.dec_stride, (size_t)(2 * METEOR_F) / sizeof(uint2) + 16));
    hw.alloc((size_t)fifo / 32 + 8);
    vsoft.alloc((size_t)max_frames * METEOR_F);
    h_ber.alloc((size_t)max_frames);
    f.max_chunks = max_frames;
    f.chunk_bits.alloc((size_t)max_frames * f.geom.bit_words + 4);
    f.start_state.alloc(max_frames + 1);
    f.redo_list.alloc(2 * (size_t)max_frames + 4);
    f.h_start.resize(max_frames + 2);
    f.rec.alloc(max_frames + 1);
    f.h_rec.alloc(max_frames + 1);
    f.tb_edges.alloc((size_t)(max_frames + 1) * f.tb_blocks);
    f.tb_list.alloc((size_t)max_frames + 2);
    f.rs_err.alloc((size_t)max_frames * METEOR_RS_I);
    f.h_rs_err.alloc((size_t)max_frames * METEOR_RS_I);
    f.frames_tmp.alloc((size_t)max_frames * METEOR_CADU);
    f.frame_dst.alloc((size_t)max_frames + 4);
    f.counters.alloc(8);
    f.h_counters.alloc(8);
    f.tables.alloc(1);
    RsTables T;
    build_rs_tables(T);
    B200_CUDA(cudaMemcpyAsync(f.tables.p, &T, sizeof(T), cudaMemcpyHostToDevice, f.stream));
    f.rec.zero(f.stream);
    B200_CUDA(cudaStreamSynchronize(f.stream)); // (T dies here)
}

std::unique_ptr<Framed> meteor_decoder(Fec &f) { return std::make_unique<Meteor>(f); }

void Meteor::reset(Fec &f)
{
    Correlated::reset(f);
    f.main_next_start = -1; // a fresh CCDecoder starts unbiased, its encoder from 0
    f.enc_state = 0;
    f.nrzm_last = 0;
    f.last_ber = 0.f;
    f.rs_avg = 0;
}

// The module loop over every frame the FIFO completes: hard bits, correlation at every even position, the frame walk, then all its frames
// at once: rotation, Viterbi27, the byte stage and RS, and the frames whose four codewords decoded into frames_out (rs_err and h_rs_err:
// RS results of the last push's frames).
void Meteor::process(Fec &f)
{
    if (!begin(f, METEOR_F))
        return;
    cudaStream_t stream = f.stream;
    const long have = f.soft_have, nwords = (have + 31) / 32 + 2, nq = (have - 64) / 2 + 1;
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    k_hard_pack<1><<<(unsigned)((nwords * 32 + 255) / 256), 256, 0, stream>>>(f.softbuf.p, have, nwords, hw.p);
    k_meteor_corr<<<(unsigned)((nq + 255) / 256), 256, 0, stream>>>(hw.p, nq, sw, score.p, bsync.p, bval.p, bidx.p);
    const Corr64Window win{hw.p, score.p, bsync.p, bval.p, bidx.p, sw};
    k_frame_walk<<<1, WALK_WARPS * 32, 0, stream>>>(win, have, METEOR_F, frames.p, (int)max_frames, walk.p);
    f.launches += 3;
    const int nf = walked(stream);
    int kept = 0;
    if (nf > 0) {
        B200_REQUIRE((size_t)(f.out_frames + nf) * METEOR_CADU <= f.frames_out.n, B200_ESTATE,
                     "%ld frames not pulled yet: pull the frames between pushes", f.out_frames);
        k_meteor_gather<<<dim3(METEOR_F / 1024, nf), 256, 0, stream>>>(f.softbuf.p, frames.p, vsoft.p);
        f.launches++;
        B200_CUDA(cudaMemcpyAsync(h_frames.p, frames.p, sizeof(WalkFrame) * nf, cudaMemcpyDeviceToHost, stream));
        viterbi_chained(f, vsoft.p, nf, h_ber.p);
        const int nrzm_next = nrzm ? f.last_raw_bit(nf - 1, METEOR_BITS) : 0;
        k_meteor_frames<<<nf, 256, 0, stream>>>(f.chunk_bits.p, f.geom.bit_words, nrzm, f.nrzm_last, f.tables.p, f.frames_tmp.p, f.rs_err.p);
        f.launches++;
        rs_usecheck_compact(f, f.frames_tmp.p, nf, METEOR_RS_I, f.frames_out.p + f.out_frames * METEOR_CADU);
        B200_CUDA(cudaMemcpyAsync(f.h_rs_err.p, f.rs_err.p, sizeof(int) * nf * METEOR_RS_I, cudaMemcpyDeviceToHost, stream));
        f.nrzm_last = nrzm_next;
    }
    f.keep_soft_tail(h_walk.p->next);
    end(f);
    finish(nf, f.soft_have);
    if (nf > 0) {
        kept = f.h_counters.p[2];
        const int *e = f.h_rs_err.p + (nf - 1) * METEOR_RS_I;
        f.rs_avg = (e[0] + e[1] + e[2] + e[3]) / 4;
        f.last_ber = ((float)h_ber.p[nf - 1] / 1024.0f) * 4.0f; // viterbi27.cpp:60-65
    }
    for (int i = 0; i < nf * METEOR_RS_I; i++) {
        const int e = f.h_rs_err.p[i];
        if (e == -1)
            f.rs_failed++;
        else
            f.rs_corrected += e;
    }
    f.out_frames += kept;
    f.total_frames += kept;
    f.total_chunks += nf;
    f.total_bits += (long)nf * METEOR_BITS;
}

long Meteor::records(const Fec &f, b200_meteor_frame *out, long cap) const
{
    B200_REQUIRE(last_nf <= cap, B200_ESTATE, "output buffer too small: need %ld records", last_nf);
    for (long k = 0; k < last_nf; k++) {
        const WalkFrame &r = h_frames.p[k];
        b200_meteor_frame &d = out[k];
        d.offset = (long)r.off;
        d.pos = r.pos;
        d.corr = (int)r.cor;
        d.phase = r.phase;
        d.swap = r.swap;
        for (int i = 0; i < METEOR_RS_I; i++)
            d.rs[i] = f.h_rs_err.p[k * METEOR_RS_I + i];
        d.ber = ((float)h_ber.p[k] / 1024.0f) * 4.0f;
    }
    return last_nf;
}

} // namespace b200

using namespace b200;

extern "C" int b200_fec_debug_meteor_frames(b200_fec *h, b200_meteor_frame *out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        Fec &f = *h->f;
        *n_out = f.framed_as<Meteor>("not a METEOR LRPT decoder in m2x_mode false").records(f, out, cap);
    });
}
