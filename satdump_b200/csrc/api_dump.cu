// Host driver of metop_dump_decoder (B200_FEC_METOP_DUMP) inside the decoder object: MetOpDumpDecoderModule::process
// (plugins/noaa_metop_support/metop/module_metop_dump_decoder.cpp:27-83) over the soft FIFO of Fec.
#include "dump.cuh"
#include "fec_host.h"

namespace b200
{

struct Dump
{
    DumpSync sw{};
    long tail_seen = -1; // FIFO bytes left by the last pass (a second process() without new bytes changes nothing)
    long max_frames = 0;
    DevBuf<uint32_t> hw;
    DevBuf<float> score, bval;
    DevBuf<int> bidx;
    DevBuf<unsigned char> bsync;
    DevBuf<LdpcFrameRec> frames;
    DevBuf<LdpcWalkOut> walk;
    LdpcWalkOut *h_walk = nullptr;
    LdpcFrameRec *h_frames = nullptr;
    long last_nf = 0; // records of the last push in h_frames (offsets made absolute) and h_rs_err
    long base = 0, resyncs = 0;
    int lock = 0, cor = 0;
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

void Fec::dump_init()
{
    B200_REQUIRE(cfg.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for the MetOp dump decoder");
    geom.chunk = DUMP_F;
    cadu_bytes = DUMP_CADU;
    cfg.cadu_size = DUMP_CADU * 8;
    cfg.constellation = B200_QPSK;
    check_device(cfg.device);
    DeviceGuard g(cfg.device);
    B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    for (cudaEvent_t *e : {&ev[0], &ev[1], &evm[0], &evm[1], &evf[0], &evf[1]}) // (the destructor destroys all six)
        B200_CUDA(cudaEventCreate(e));
    dump = new Dump();
    Dump &D = *dump;
    for (int p = 0; p < 4; p++) {
        D.sw.w[p] = rotate_64(0x1acffc1du, p);
        D.sw.w[4 + p] = rotate_64(swap_iq(0x1acffc1du) ^ 0xffffffffu, p); // (the module's 0xFFFFFFFFFF truncated to 32 bits)
    }
    const long fifo = cfg.max_soft + 2L * DUMP_F;
    softbuf.alloc((size_t)fifo);
    dec.alloc((size_t)(2 * DUMP_F) / sizeof(uint2) + 16); // scratch of keep_soft_tail
    D.hw.alloc((size_t)fifo / 32 + 8);
    D.score.alloc((size_t)fifo / 2);
    D.bsync.alloc((size_t)fifo / 2);
    D.bval.alloc((size_t)fifo / 64 + 2);
    D.bidx.alloc((size_t)fifo / 64 + 2);
    D.max_frames = fifo / DUMP_F + 2;
    D.frames.alloc((size_t)D.max_frames);
    D.walk.alloc(1);
    rs_err.alloc((size_t)D.max_frames * DUMP_RS_I);
    max_frames_push = D.max_frames;
    frames_out.alloc((size_t)(2 * D.max_frames + 4) * DUMP_CADU);
    tables.alloc(1);
    RsTables T;
    build_rs_tables(T);
    B200_CUDA(cudaMemcpyAsync(tables.p, &T, sizeof(T), cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMallocHost((void **)&D.h_walk, sizeof(LdpcWalkOut)));
    B200_CUDA(cudaMallocHost((void **)&D.h_frames, sizeof(LdpcFrameRec) * D.max_frames));
    B200_CUDA(cudaMallocHost((void **)&h_rs_err, sizeof(int) * D.max_frames * DUMP_RS_I));
    B200_CUDA(cudaStreamSynchronize(stream)); // (T dies here)
}

void Fec::dump_free()
{
    if (!dump)
        return;
    for (void *p : {(void *)dump->h_walk, (void *)dump->h_frames})
        if (p)
            cudaFreeHost(p);
    delete dump;
    dump = nullptr;
}

void Fec::dump_reset()
{
    soft_have = 0;
    out_frames = 0;
    dump->tail_seen = -1;
    dump->base = 0;
    dump->last_nf = 0;
    dump->lock = dump->cor = 0;
}

// The module loop over every frame the FIFO completes: hard bits, correlation at every even position, the frame walk, then all its frames
// at once into frames_out. The bytes behind the walk's next window stay in the FIFO; a call that finds no new bytes behind them has
// nothing to do.
void Fec::dump_process()
{
    Dump &D = *dump;
    if (soft_have == D.tail_seen)
        return;
    D.last_nf = 0;
    if (soft_have < DUMP_F) {
        D.tail_seen = soft_have;
        return;
    }
    const long have = soft_have, nwords = (have + 31) / 32 + 2, nq = (have - 32) / 2 + 1;
    B200_CUDA(cudaEventRecord(ev[0], stream));
    k_dump_pack<<<(unsigned)((nwords * 32 + 255) / 256), 256, 0, stream>>>(softbuf.p, have, nwords, D.hw.p);
    k_dump_corr<<<(unsigned)((nq + 255) / 256), 256, 0, stream>>>(D.hw.p, nq, D.sw, D.score.p, D.bsync.p, D.bval.p, D.bidx.p);
    k_dump_walk<<<1, DUMP_WALK_WARPS * 32, 0, stream>>>(D.hw.p, D.score.p, D.bsync.p, D.bval.p, D.bidx.p, D.sw, have, D.frames.p,
                                                         (int)D.max_frames, D.walk.p);
    launches += 3;
    B200_CUDA(cudaMemcpyAsync(D.h_walk, D.walk.p, sizeof(LdpcWalkOut), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    const int nf = D.h_walk->nf;
    if (nf > 0) {
        B200_REQUIRE((size_t)(out_frames + nf) * DUMP_CADU <= frames_out.n, B200_ESTATE, "%ld frames not pulled yet: pull the frames between pushes",
                     out_frames);
        k_dump_frames<<<nf, 256, 0, stream>>>(softbuf.p, D.frames.p, tables.p, frames_out.p + out_frames * DUMP_CADU, rs_err.p);
        launches++;
        B200_CUDA(cudaMemcpyAsync(D.h_frames, D.frames.p, sizeof(LdpcFrameRec) * nf, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaMemcpyAsync(h_rs_err, rs_err.p, sizeof(int) * nf * DUMP_RS_I, cudaMemcpyDeviceToHost, stream));
    }
    keep_soft_tail(D.h_walk->next);
    B200_CUDA(cudaEventRecord(ev[1], stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&t_vit, ev[0], ev[1]);
    for (int k = 0; k < nf; k++) {
        LdpcFrameRec &r = D.h_frames[k];
        r.off += D.base;
        D.resyncs += r.pos != 0;
        for (int i = 0; i < DUMP_RS_I; i++) {
            const int e = h_rs_err[k * DUMP_RS_I + i];
            if (e == -1)
                rs_failed++;
            else
                rs_corrected += e;
        }
    }
    if (nf > 0) {
        D.lock = D.h_frames[nf - 1].pos == 0;
        D.cor = (int)D.h_frames[nf - 1].cor;
    }
    D.last_nf = nf;
    D.base += D.h_walk->next;
    D.tail_seen = soft_have;
    out_frames += nf;
    total_frames += nf;
    total_chunks += nf;
    total_bits += (long)nf * DUMP_CADU * 8;
}

void Fec::dump_stats(b200_fec_stats *o)
{
    o->correlator_lock = dump->lock;
    o->correlator_corr = (float)dump->cor;
    o->ldpc_resyncs = dump->resyncs;
}

long Fec::dump_frames(b200_dump_frame *out, long cap)
{
    B200_REQUIRE(dump, B200_EINVAL, "not a MetOp dump decoder");
    B200_REQUIRE(dump->last_nf <= cap, B200_ESTATE, "output buffer too small: need %ld records", dump->last_nf);
    for (long k = 0; k < dump->last_nf; k++) {
        const LdpcFrameRec &r = dump->h_frames[k];
        b200_dump_frame &d = out[k];
        d.offset = (long)r.off;
        d.pos = r.pos;
        d.corr = (int)r.cor;
        d.phase = r.phase;
        d.swap = r.swap;
        for (int i = 0; i < DUMP_RS_I; i++)
            d.rs[i] = h_rs_err[k * DUMP_RS_I + i];
    }
    return dump->last_nf;
}

} // namespace b200
