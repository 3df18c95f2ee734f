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
    Viterbi vit;
    FrameStage fs;              // the RS tables, results and rs_usecheck of k_meteor_frames
    int nrzm = 0, nrzm_last = 0;
    float ber = 0.f;            // Viterbi27's d_ber (0 before the first frame)

    explicit Meteor(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
    void stats(b200_fec_stats *o) override;
    long records(b200_meteor_frame *out, long cap) const; // of the last push
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
} // namespace

Meteor::Meteor(Fec &f)
{
    B200_REQUIRE(f.cfg.max_soft <= (1L << 28), B200_EINVAL, "max_soft must be <= 2^28 for the METEOR LRPT decoder");
    nrzm = f.cfg.diff_decode != 0;
    f.chunk = METEOR_F;
    f.cadu_bytes = METEOR_CADU;
    vit.spec_steps = VIT_SPEC_STEPS_12;
    const uint64_t word = nrzm ? 0xfc4ef4fd0cc2df89ull : 0xfca2b63db00d9794ull;
    for (int p = 0; p < 4; p++) {
        sw.w[p] = rotate_64(word, p);
        sw.w[4 + p] = rotate_64(swap_iq(word) ^ ~0ull, p);
    }
    check_device(f.cfg.device);
    DeviceGuard g(f.cfg.device);
    const long fifo = f.cfg.max_soft + 2L * METEOR_F;
    alloc(fifo / 2, fifo / METEOR_F + 2); // scores at the even positions
    f.open(METEOR_F, max_frames);
    hw.alloc((size_t)fifo / 32 + 8);
    vsoft.alloc((size_t)max_frames * METEOR_F);
    h_ber.alloc((size_t)max_frames);
    // Viterbi27(8192) (common/codings/viterbi/viterbi27.cpp): frame size, and the BER test re-encodes 512 bits and compares 1024 symbols
    VitGeom geom{};
    geom.chunk = METEOR_F;
    geom.F = METEOR_BITS;
    geom.ber_bits = 512;
    geom.ber_syms = 1024;
    vit.alloc(f, geom, max_frames); // (the decisions of every frame of a push)
    fs.alloc(f, max_frames, METEOR_RS_I, true);
}

std::unique_ptr<Decoder> meteor_decoder(Fec &f) { return std::make_unique<Meteor>(f); }

void Meteor::reset(Fec &f)
{
    Correlated::reset(f);
    vit.main_next_start = -1; // a fresh CCDecoder starts unbiased, its encoder from 0
    vit.enc_state = 0;
    nrzm_last = 0;
    ber = 0.f;
}

void Meteor::stats(b200_fec_stats *o)
{
    Correlated::stats(o);
    o->viterbi_ber = ber;
    vit.stats(o);
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
        vit.chained(f, vsoft.p, nf, h_ber.p);
        const int nrzm_next = nrzm ? last_raw_bit(f, vit.chunk_bits.p, vit.geom.bit_words, nf - 1, METEOR_BITS) : 0;
        k_meteor_frames<<<nf, 256, 0, stream>>>(vit.chunk_bits.p, vit.geom.bit_words, nrzm, nrzm_last, fs.tables.p, fs.frames_tmp.p, fs.rs_err.p);
        f.launches++;
        fs.usecheck(f, fs.frames_tmp.p, nf, METEOR_RS_I, f.frames_out.p + f.out_frames * METEOR_CADU);
        B200_CUDA(cudaMemcpyAsync(fs.h_rs_err.p, fs.rs_err.p, sizeof(int) * nf * METEOR_RS_I, cudaMemcpyDeviceToHost, stream));
        nrzm_last = nrzm_next;
    }
    f.keep_soft_tail(h_walk.p->next);
    end(f);
    finish(nf, f.soft_have);
    if (nf > 0) {
        kept = fs.h_counters.p[2];
        const int *e = fs.h_rs_err.p + (nf - 1) * METEOR_RS_I;
        f.rs_avg = (e[0] + e[1] + e[2] + e[3]) / 4;
        ber = ((float)h_ber.p[nf - 1] / 1024.0f) * 4.0f; // viterbi27.cpp:60-65
    }
    fs.count_rs(f, nf, METEOR_RS_I);
    f.out_frames += kept;
    f.total_frames += kept;
    f.total_chunks += nf;
    f.total_bits += (long)nf * METEOR_BITS;
}

long Meteor::records(b200_meteor_frame *out, long cap) const
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
            d.rs[i] = fs.h_rs_err.p[k * METEOR_RS_I + i];
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
        *n_out = h->f->decoder_as<Meteor>("not a METEOR LRPT decoder in m2x_mode false").records(out, cap);
    });
}
