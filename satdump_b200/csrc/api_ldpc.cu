// Host driver of ccsds_ldpc_decoder (B200_FEC_LDPC) inside the decoder object: CCSDSLDPCDecoderModule::process
// (src-core/pipeline/modules/ccsds/module_ccsds_ldpc_decoder.cpp:134-277) for ldpc_rate "7/8", over the soft FIFO of Fec.
#include "fec_host.h"
#include "ldpc.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

#include "ldpc_c2_table.inc"

namespace b200
{

struct Ldpc
{
    int constellation = 0, nsync = 0, nlevels = 0;
    bool derandomize = true, internal = false;
    long tail_seen = -1; // FIFO bytes left by the last pass (a second process() without new bytes changes nothing)
    LdpcSync sw{};
    long max_frames = 0;
    DevBuf<float> score, bval;
    DevBuf<int> bidx, level_ptr;
    DevBuf<unsigned char> bsync, pn;
    DevBuf<LdpcFrameRec> frames;
    DevBuf<LdpcWalkOut> walk;
    DevBuf<int8_t> vn;
    DevBuf<uint8_t> cadu_tmp; // internal_stream: the codewords' CADUs, whose info bits go to the bit FIFO
    DevBuf<uint16_t> cols, level_rows;
    LdpcWalkOut *h_walk = nullptr;
    LdpcFrameRec *h_frames = nullptr;
    long last_nf = 0; // records of the last push in h_frames (offsets made absolute)
    // stream state and the module's statistics
    long base = 0, resyncs = 0;
    int lock = 0, corr = 0;
    float cor = 0.f;
    cudaEvent_t ev[6]{};
    float t_ms[5]{}; // last push: correlation, walk, gather, decode + repack, and the whole push
};

namespace
{
// H row by row (make_ccsds.cpp:407-430: row block 0's 511 rows, then row block 1's), the 32 columns of a row ascending
std::vector<uint16_t> c2_rows()
{
    std::vector<uint16_t> cols(LDPC_ROWS * LDPC_DEG);
    for (int y = 0; y < LDPC_C2_BY; y++)
        for (int r = 0; r < LDPC_C2_CIRC; r++) {
            uint16_t *row = &cols[(y * LDPC_C2_CIRC + r) * LDPC_DEG];
            for (int x = 0; x < LDPC_C2_BX; x++) {
                int a = (ldpc_c2_offsets[y][x][0] + r) % LDPC_C2_CIRC, b = (ldpc_c2_offsets[y][x][1] + r) % LDPC_C2_CIRC;
                if (a > b) std::swap(a, b);
                row[2 * x] = (uint16_t)(LDPC_C2_CIRC * x + a);
                row[2 * x + 1] = (uint16_t)(LDPC_C2_CIRC * x + b);
            }
        }
    return cols;
}

// The level schedule of `iterations` x rows 0 .. R-1 (see k_ldpc_decode): ptr[L] .. ptr[L+1] index the rows of level L in `rows`.
void level_schedule(const std::vector<uint16_t> &cols, int iterations, std::vector<int> &ptr, std::vector<uint16_t> &rows)
{
    std::vector<int> last(LDPC_VN, -1);
    std::vector<std::vector<uint16_t>> levels;
    for (int it = 0; it < iterations; it++)
        for (int r = 0; r < LDPC_ROWS; r++) {
            int L = 0;
            for (int k = 0; k < LDPC_DEG; k++)
                L = std::max(L, last[cols[r * LDPC_DEG + k]] + 1);
            for (int k = 0; k < LDPC_DEG; k++)
                last[cols[r * LDPC_DEG + k]] = L;
            if ((int)levels.size() <= L)
                levels.resize(L + 1);
            levels[L].push_back((uint16_t)r);
        }
    ptr.assign(1, 0);
    rows.clear();
    for (auto &l : levels) {
        rows.insert(rows.end(), l.begin(), l.end());
        ptr.push_back((int)rows.size());
    }
}

// CorrelatorGeneric's syncword tables for the ASM 0x1ACFFC1D (generic_correlator.cpp:7-64): modulate_soft (bit 1 -> 1.0f, 0 -> -1.0f),
// then rotate_float_buf (:137-143) with its float expressions: the angle deg * 0.01745329 evaluated in double and stored as float,
// cosf / sinf of it, and the complex product (a c - b s, b c + a s), each operation rounded (no contraction on the host).
void rotate_table(float *w, float deg)
{
    const float ph = deg * 0.01745329;
    const float c = cosf(ph), s = sinf(ph);
    for (int i = 0; i < LDPC_ASM / 2; i++) {
        const float re = w[2 * i], im = w[2 * i + 1];
        w[2 * i] = (re * c) - (im * s);
        w[2 * i + 1] = (im * c) + (re * s);
    }
}
int syncwords(int constellation, LdpcSync &sw)
{
    unsigned char bits[LDPC_ASM];
    for (int i = 0; i < LDPC_ASM; i++)
        bits[i] = (0x1acffc1du >> (31 - i)) & 1;
    auto modulate = [&](float *w) {
        for (int i = 0; i < LDPC_ASM; i++)
            w[i] = bits[i] ? 1.0f : -1.0f;
    };
    if (constellation == B200_BPSK) {
        modulate(sw.w[0]);
        modulate(sw.w[1]);
        rotate_table(sw.w[1], 180);
        return 2;
    }
    if (constellation == B200_QPSK) {
        for (int s = 0; s < 4; s++) {
            modulate(sw.w[s]);
            if (s)
                rotate_table(sw.w[s], 90.0f * s);
        }
        return 4;
    }
    // OQPSK: tables 2 and 3 are the syncword with Q one symbol late (the wrong rail delayed)
    modulate(sw.w[0]);
    modulate(sw.w[1]);
    unsigned char last = 0;
    for (int i = 0; i < LDPC_ASM / 2; i++) {
        const unsigned char back = bits[2 * i + 1];
        bits[2 * i + 1] = last;
        last = back;
    }
    modulate(sw.w[2]);
    modulate(sw.w[3]);
    rotate_table(sw.w[0], 90);
    rotate_table(sw.w[1], 270);
    rotate_table(sw.w[3], 180);
    return 4;
}
} // namespace

void ccsds_pn_bits(unsigned char *pn)
{
    uint8_t reg = 0xFF;
    for (int i = 0; i < 255; i++) {
        pn[i] = reg >> 7;
        const uint8_t nb = ((reg >> 7) ^ (reg >> 4) ^ (reg >> 2) ^ reg) & 1;
        reg = (uint8_t)((reg << 1) | nb);
    }
}

void frame_walk(const float *score, const unsigned char *best_sync, const float *bval, const int *bidx, long have, int F, int npos,
                int constellation, LdpcFrameRec *frames, int max_frames, LdpcWalkOut *out, cudaStream_t stream)
{
    k_ldpc_walk<<<1, LDPC_WALK_WARPS * 32, 0, stream>>>(score, best_sync, bval, bidx, have, F, npos, constellation, frames, max_frames, out);
}

// Everything this build does not cover is refused by name before the device is touched.
void Fec::ldpc_init()
{
    const b200_fec_cfg &c = cfg;
    B200_REQUIRE(!c.ldpc2, B200_EUNSUPPORTED, "ldpc2 (the labrador LDPC decoder) is not built");
    B200_REQUIRE(c.ldpc_rate != 1 && c.ldpc_rate != 2 && c.ldpc_rate != 4, B200_EUNSUPPORTED,
                 "ldpc_rate 1/2, 2/3 and 4/5 (the AR4JA codes, ldpc_block_size) are not built: only 7/8 (C2)");
    B200_REQUIRE(c.ldpc_rate == 7, B200_EINVAL, "Invalid LDPC code rate %d (7 = \"7/8\")", c.ldpc_rate);
    B200_REQUIRE(!(c.internal_stream && c.internal_cadu_size % 8 != 0), B200_EUNSUPPORTED,
                 "internal_cadu_size %d is not a multiple of 8 (frame padding is not built)", c.internal_cadu_size);
    B200_REQUIRE(!c.internal_stream || (c.internal_cadu_size >= 64 && c.internal_cadu_size <= 65536), B200_EINVAL,
                 "internal_cadu_size out of range (64..65536)");
    B200_REQUIRE(c.constellation != B200_8PSK, B200_EUNSUPPORTED, "8PSK is not built for the LDPC decoder");
    B200_REQUIRE(c.constellation == B200_BPSK || c.constellation == B200_QPSK || c.constellation == B200_OQPSK, B200_EINVAL,
                 "CCSDS LDPC Decoder : invalid constellation type!");
    B200_REQUIRE(c.ldpc_iterations >= 0 && c.ldpc_iterations <= 1000, B200_EINVAL, "ldpc_iterations out of range (0..1000)");
    B200_REQUIRE(c.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for the LDPC decoder");
    geom.chunk = LDPC_F;
    cadu_bytes = c.internal_stream ? c.internal_cadu_size / 8 : LDPC_CADU;
    cfg.cadu_size = c.internal_stream ? c.internal_cadu_size : LDPC_CADU * 8;
    const bool derand = c.derandomize != 0;
    if (c.internal_stream) { // BPSK_CCSDS_Deframer(internal_cadu_size, internal_asm) (:100-113): plain frames, no RS, no derandomiser
        cfg.rs_i = 0;
        cfg.derandomize = cfg.derand_after_rs = cfg.rs_usecheck = 0;
        cfg.nrzm = 0;
        if (cfg.asm_sync == 0)
            cfg.asm_sync = 0x1ACFFC1D;
        st_synced = 12;
    }
    check_device(c.device);
    DeviceGuard g(c.device);
    B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    for (cudaEvent_t *e : {&ev[0], &ev[1], &evm[0], &evm[1], &evf[0], &evf[1]}) // (the destructor destroys all six)
        B200_CUDA(cudaEventCreate(e));
    ldpc = new Ldpc();
    Ldpc &L = *ldpc;
    for (auto &e : L.ev)
        B200_CUDA(cudaEventCreate(&e));
    L.constellation = c.constellation;
    L.derandomize = derand;
    L.internal = c.internal_stream != 0;
    L.nsync = syncwords(c.constellation, L.sw);
    const long fifo = c.max_soft + 2L * LDPC_F;
    softbuf.alloc((size_t)fifo);
    dec.alloc((size_t)(2 * LDPC_F) / sizeof(uint2) + 16); // scratch of keep_soft_tail
    L.score.alloc((size_t)fifo);
    L.bsync.alloc((size_t)fifo);
    L.bval.alloc((size_t)fifo / 32 + 2);
    L.bidx.alloc((size_t)fifo / 32 + 2);
    L.max_frames = fifo / LDPC_F + 2;
    L.frames.alloc((size_t)L.max_frames);
    L.walk.alloc(1);
    L.vn.alloc((size_t)L.max_frames * LDPC_VN);
    if (L.internal) {
        L.cadu_tmp.alloc((size_t)L.max_frames * LDPC_CADU);
        deframer_storage(L.max_frames * (long)LDPC_INFO_BITS);
    } else {
        max_frames_push = L.max_frames;
        frames_out.alloc((size_t)(2 * L.max_frames + 4) * LDPC_CADU);
    }
    const std::vector<uint16_t> cols = c2_rows();
    std::vector<int> ptr;
    std::vector<uint16_t> rows;
    level_schedule(cols, c.ldpc_iterations, ptr, rows);
    L.nlevels = (int)ptr.size() - 1;
    L.cols.alloc(cols.size());
    L.level_ptr.alloc(ptr.size());
    L.level_rows.alloc(std::max<size_t>(rows.size(), 1));
    unsigned char pnb[255];
    ccsds_pn_bits(pnb);
    L.pn.alloc(256);
    B200_CUDA(cudaMemcpyAsync(L.cols.p, cols.data(), cols.size() * sizeof(uint16_t), cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMemcpyAsync(L.level_ptr.p, ptr.data(), ptr.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
    if (!rows.empty())
        B200_CUDA(cudaMemcpyAsync(L.level_rows.p, rows.data(), rows.size() * sizeof(uint16_t), cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMemcpyAsync(L.pn.p, pnb, 255, cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMallocHost((void **)&L.h_walk, sizeof(LdpcWalkOut)));
    B200_CUDA(cudaMallocHost((void **)&L.h_frames, sizeof(LdpcFrameRec) * L.max_frames));
    B200_CUDA(cudaStreamSynchronize(stream)); // (the host vectors above die here)
}

void Fec::ldpc_free()
{
    if (!ldpc)
        return;
    for (auto &e : ldpc->ev)
        if (e)
            cudaEventDestroy(e);
    if (ldpc->h_walk)
        cudaFreeHost(ldpc->h_walk);
    if (ldpc->h_frames)
        cudaFreeHost(ldpc->h_frames);
    delete ldpc;
    ldpc = nullptr;
}

void Fec::ldpc_reset()
{
    if (ldpc->internal) {
        start_stream(64); // the bit FIFO and the deframer
        B200_CUDA(cudaStreamSynchronize(stream));
    }
    soft_have = 0;
    out_frames = 0;
    ldpc->tail_seen = -1;
    ldpc->base = 0;
    ldpc->last_nf = 0;
    ldpc->lock = ldpc->corr = 0;
    ldpc->cor = 0.f;
}

// The module loop over every frame the FIFO completes: correlation at every position, the frame walk, then gather, decode and repack of
// all its frames at once (internal_stream: their info bits through the bit FIFO and the deframer). The bytes behind the walk's next window
// stay in the FIFO; a call that finds no new bytes behind them has nothing to do.
void Fec::ldpc_process()
{
    Ldpc &L = *ldpc;
    if (soft_have == L.tail_seen)
        return;
    L.last_nf = 0;
    for (float &t : L.t_ms)
        t = 0;
    last_bits0 = last_nbits = 0;
    t_frames = 0;
    if (soft_have < LDPC_F) {
        L.tail_seen = soft_have;
        return;
    }
    if (L.internal)
        compact_fifo(false);
    const long have = soft_have, npos = have - (LDPC_ASM - 1);
    B200_CUDA(cudaEventRecord(L.ev[0], stream));
    k_ldpc_corr<<<(unsigned)((npos + 255) / 256), 256, 0, stream>>>(softbuf.p, npos, L.sw, L.nsync, L.score.p, L.bsync.p, L.bval.p, L.bidx.p);
    B200_CUDA(cudaEventRecord(L.ev[1], stream));
    frame_walk(L.score.p, L.bsync.p, L.bval.p, L.bidx.p, have, LDPC_F, LDPC_NPOS, L.constellation, L.frames.p, (int)L.max_frames, L.walk.p, stream);
    B200_CUDA(cudaEventRecord(L.ev[2], stream));
    launches += 2;
    B200_CUDA(cudaMemcpyAsync(L.h_walk, L.walk.p, sizeof(LdpcWalkOut), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    const int nf = L.h_walk->nf;
    if (nf > 0) {
        B200_REQUIRE(L.internal || (size_t)(out_frames + nf) * LDPC_CADU <= frames_out.n, B200_ESTATE,
                     "%ld frames not pulled yet: pull the frames between pushes", out_frames);
        k_ldpc_gather<<<nf, 256, 0, stream>>>(softbuf.p, L.frames.p, L.constellation == B200_OQPSK, L.derandomize ? L.pn.p : nullptr, L.vn.p);
        B200_CUDA(cudaEventRecord(L.ev[3], stream));
        const int smem = ((LDPC_VN * 2 + 15) & ~15) + LDPC_ROWS * (int)sizeof(LdpcRowMsg);
        uint8_t *cadu = L.internal ? L.cadu_tmp.p : frames_out.p + out_frames * LDPC_CADU;
        k_ldpc_decode<<<nf, LDPC_DEC_THREADS, smem, stream>>>(L.vn.p, L.cols.p, L.level_ptr.p, L.level_rows.p, L.nlevels, L.frames.p, cadu);
        launches += 2;
        B200_CUDA(cudaMemcpyAsync(L.h_frames, L.frames.p, sizeof(LdpcFrameRec) * nf, cudaMemcpyDeviceToHost, stream));
        if (L.internal) { // :233-242: deframer->work(first 7136 decoded bits) of every codeword, in stream order
            const long new_bits = (long)nf * LDPC_INFO_BITS;
            const long words = (new_bits + 63) / 32;
            k_ldpc_append<<<(unsigned)std::min<long>((words + 255) / 256, 132 * 8), 256, 0, stream>>>(cadu, nf, fifo.p, fifo_bits);
            launches++;
            last_bits0 = fifo_bits;
            last_nbits = new_bits;
            deframe_and_rs(new_bits); // (synchronises the stream)
        }
        B200_CUDA(cudaEventRecord(L.ev[4], stream));
    }
    keep_soft_tail(L.h_walk->next);
    B200_CUDA(cudaEventRecord(L.ev[5], stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&L.t_ms[0], L.ev[0], L.ev[1]);
    cudaEventElapsedTime(&L.t_ms[1], L.ev[1], L.ev[2]);
    if (nf > 0) {
        cudaEventElapsedTime(&L.t_ms[2], L.ev[2], L.ev[3]);
        cudaEventElapsedTime(&L.t_ms[3], L.ev[3], L.ev[4]);
    }
    cudaEventElapsedTime(&L.t_ms[4], L.ev[0], L.ev[5]);
    t_vit = L.t_ms[4];
    for (int k = 0; k < nf; k++) {
        LdpcFrameRec &r = L.h_frames[k];
        r.off += L.base;
        L.resyncs += r.pos != 0;
    }
    if (nf > 0) {
        const LdpcFrameRec &r = L.h_frames[nf - 1];
        L.lock = r.pos == 0;
        L.cor = r.cor;
        L.corr = r.corr;
    }
    L.last_nf = nf;
    L.base += L.h_walk->next;
    L.tail_seen = soft_have;
    if (!L.internal) { // (internal_stream: deframe_and_rs counted the inner frames)
        out_frames += nf;
        total_frames += nf;
    }
    total_chunks += nf;
    total_bits += (long)nf * LDPC_CW;
}

void Fec::ldpc_stats(b200_fec_stats *o)
{
    o->correlator_lock = ldpc->lock;
    o->correlator_corr = ldpc->cor;
    o->ldpc_corr = ldpc->corr;
    o->ldpc_resyncs = ldpc->resyncs;
}

long Fec::ldpc_frames(b200_ldpc_frame *out, long cap)
{
    B200_REQUIRE(ldpc, B200_EINVAL, "not an LDPC decoder");
    B200_REQUIRE(ldpc->last_nf <= cap, B200_ESTATE, "output buffer too small: need %ld records", ldpc->last_nf);
    for (long k = 0; k < ldpc->last_nf; k++) {
        const LdpcFrameRec &r = ldpc->h_frames[k];
        out[k] = b200_ldpc_frame{(long)r.off, r.pos, r.cor, r.phase, r.swap, r.corr};
    }
    return ldpc->last_nf;
}

void Fec::ldpc_timing(float *ms, int n)
{
    for (int k = 0; k < n && k < 5; k++)
        ms[k] = ldpc ? ldpc->t_ms[k] : 0.f;
}

} // namespace b200
