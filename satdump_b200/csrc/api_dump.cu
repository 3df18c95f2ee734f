// Host driver of metop_dump_decoder (B200_FEC_METOP_DUMP) inside the decoder object: MetOpDumpDecoderModule::process
// (plugins/noaa_metop_support/metop/module_metop_dump_decoder.cpp:27-83) over the soft FIFO of Fec.
#include "dump.cuh"
#include "fec_host.h"

namespace b200
{

struct Dump : Framed
{
    DumpSync sw{};
    DevBuf<uint32_t> hw;

    explicit Dump(Fec &f);
    void process(Fec &f) override;
};

namespace
{
// correlator32.cpp:3-42
uint32_t rotate_64(uint32_t word, int p)
{
    const uint32_t i = word & 0xaaaaaaaau, q = word & 0x55555555u;
    switch (p) {
    case 1: word = ((i ^ 0xaaaaaaaau) >> 1) | (q << 1); break;
    case 2: word = word ^ 0xffffffffu; break;
    case 3: word = (i >> 1) | ((q ^ 0x55555555u) << 1); break;
    default: break;
    }
    return ((word & 0x55555555u) << 1) | ((word & 0xaaaaaaaau) >> 1);
}
uint32_t swap_iq(uint32_t w) { return ((w & 0xaaaaaaaau) >> 1) | ((w & 0x55555555u) << 1); }
} // namespace

Dump::Dump(Fec &f)
{
    B200_REQUIRE(f.cfg.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for the MetOp dump decoder");
    f.geom.chunk = DUMP_F;
    f.cadu_bytes = DUMP_CADU;
    f.cfg.cadu_size = DUMP_CADU * 8;
    f.cfg.constellation = B200_QPSK;
    for (int p = 0; p < 4; p++) {
        sw.w[p] = rotate_64(0x1acffc1du, p);
        sw.w[4 + p] = rotate_64(swap_iq(0x1acffc1du) ^ 0xffffffffu, p); // (the module's 0xFFFFFFFFFF truncated to 32 bits)
    }
    check_device(f.cfg.device);
    DeviceGuard g(f.cfg.device);
    const long fifo = f.cfg.max_soft + 2L * DUMP_F;
    alloc(fifo / 2, fifo / DUMP_F + 2); // scores at the even positions
    f.framed_storage(DUMP_F, max_frames);
    hw.alloc((size_t)fifo / 32 + 8);
    f.rs_err.alloc((size_t)max_frames * DUMP_RS_I);
    f.h_rs_err.alloc((size_t)max_frames * DUMP_RS_I);
    f.tables.alloc(1);
    RsTables T;
    build_rs_tables(T);
    B200_CUDA(cudaMemcpyAsync(f.tables.p, &T, sizeof(T), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream)); // (T dies here)
}

std::unique_ptr<Framed> dump_decoder(Fec &f) { return std::make_unique<Dump>(f); }

// The module loop over every frame the FIFO completes: hard bits, correlation at every even position, the frame walk, then all its frames
// at once into frames_out (rs_err and h_rs_err: RS results of the last push's frames).
void Dump::process(Fec &f)
{
    if (!begin(f, DUMP_F))
        return;
    cudaStream_t stream = f.stream;
    const long have = f.soft_have, nwords = (have + 31) / 32 + 2, nq = (have - 32) / 2 + 1;
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    k_hard_pack<0><<<(unsigned)((nwords * 32 + 255) / 256), 256, 0, stream>>>(f.softbuf.p, have, nwords, hw.p);
    k_dump_corr<<<(unsigned)((nq + 255) / 256), 256, 0, stream>>>(hw.p, nq, sw, score.p, bsync.p, bval.p, bidx.p);
    const DumpWindow win{hw.p, score.p, bsync.p, bval.p, bidx.p, sw};
    k_frame_walk<<<1, WALK_WARPS * 32, 0, stream>>>(win, have, DUMP_F, frames.p, (int)max_frames, walk.p);
    f.launches += 3;
    const int nf = walked(stream);
    if (nf > 0) {
        B200_REQUIRE((size_t)(f.out_frames + nf) * DUMP_CADU <= f.frames_out.n, B200_ESTATE,
                     "%ld frames not pulled yet: pull the frames between pushes", f.out_frames);
        k_dump_frames<<<nf, 256, 0, stream>>>(f.softbuf.p, frames.p, f.tables.p, f.frames_out.p + f.out_frames * DUMP_CADU, f.rs_err.p);
        f.launches++;
        B200_CUDA(cudaMemcpyAsync(h_frames.p, frames.p, sizeof(WalkFrame) * nf, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaMemcpyAsync(f.h_rs_err.p, f.rs_err.p, sizeof(int) * nf * DUMP_RS_I, cudaMemcpyDeviceToHost, stream));
    }
    f.keep_soft_tail(h_walk.p->next);
    B200_CUDA(cudaEventRecord(f.ev[1], stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&f.t_vit, f.ev[0], f.ev[1]);
    finish(nf, f.soft_have);
    for (int i = 0; i < nf * DUMP_RS_I; i++) {
        const int e = f.h_rs_err.p[i];
        if (e == -1)
            f.rs_failed++;
        else
            f.rs_corrected += e;
    }
    f.out_frames += nf;
    f.total_frames += nf;
    f.total_chunks += nf;
    f.total_bits += (long)nf * DUMP_CADU * 8;
}

long Fec::dump_frames(b200_dump_frame *out, long cap)
{
    const Dump &D = framed_as<Dump>("not a MetOp dump decoder");
    B200_REQUIRE(D.last_nf <= cap, B200_ESTATE, "output buffer too small: need %ld records", D.last_nf);
    for (long k = 0; k < D.last_nf; k++) {
        const WalkFrame &r = D.h_frames.p[k];
        b200_dump_frame &d = out[k];
        d.offset = (long)r.off;
        d.pos = r.pos;
        d.corr = (int)r.cor;
        d.phase = r.phase;
        d.swap = r.swap;
        for (int i = 0; i < DUMP_RS_I; i++)
            d.rs[i] = h_rs_err.p[k * DUMP_RS_I + i];
    }
    return D.last_nf;
}

} // namespace b200
