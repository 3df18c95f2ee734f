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

struct Ldpc : Correlated
{
    int constellation = 0, nsync = 0, nlevels = 0;
    bool derandomize = true, internal = false;
    int corr = 0; // ldpc_corr of the last frame
    LdpcSync sw{};
    DevBuf<int> level_ptr;
    DevBuf<unsigned char> pn;
    DevBuf<int8_t> vn;
    DevBuf<uint8_t> cadu_tmp; // internal_stream: the codewords' CADUs, whose info bits go to the bit FIFO
    DevBuf<uint16_t> cols, level_rows;
    Events<6> ev; // t_ms: correlation, walk, gather, decode + repack, and the whole push
    Deframer defr;  // internal_stream: the bit FIFO of the info bits ...
    FrameStage fs;  // ... and its frame stage

    explicit Ldpc(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
    void stats(b200_fec_stats *o) override;
    const Deframer *deframer() const override { return &defr; }
    long records(b200_ldpc_frame *out, long cap) const; // of the last push
    void timing(float *ms, int n) const;
};

// Everything this build does not cover is refused by name before the device is touched.
Ldpc::Ldpc(Fec &f)
{
    const b200_fec_cfg &c = f.cfg;
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
    derandomize = c.derandomize != 0; // (before internal_stream clears it for the deframer stage)
    f.chunk = LDPC_F;
    f.cadu_bytes = c.internal_stream ? c.internal_cadu_size / 8 : LDPC_CADU;
    f.cfg.cadu_size = c.internal_stream ? c.internal_cadu_size : LDPC_CADU * 8;
    if (c.internal_stream) { // BPSK_CCSDS_Deframer(internal_cadu_size, internal_asm) (:100-113): plain frames, no RS, no derandomiser
        f.cfg.rs_i = 0;
        f.cfg.derandomize = f.cfg.derand_after_rs = f.cfg.rs_usecheck = 0;
        f.cfg.nrzm = 0;
        if (f.cfg.asm_sync == 0)
            f.cfg.asm_sync = 0x1ACFFC1D;
    }
    constellation = c.constellation;
    internal = c.internal_stream != 0;
    nsync = syncwords(c.constellation, sw);
    check_device(c.device);
    DeviceGuard g(c.device);
    const long fifo = c.max_soft + 2L * LDPC_F;
    alloc(fifo, fifo / LDPC_F + 2);
    const long max_bits = max_frames * (long)LDPC_INFO_BITS; // internal_stream: the bit FIFO's new bits a push
    f.open(LDPC_F, internal ? Deframer::frames_cap(max_bits, f.cfg.cadu_size) : max_frames);
    ev.create();
    vn.alloc((size_t)max_frames * LDPC_VN);
    if (internal) {
        cadu_tmp.alloc((size_t)max_frames * LDPC_CADU);
        defr.alloc(f, max_bits, f.cfg.cadu_size, f.cfg.asm_sync, 12);
        fs.alloc(f, Deframer::frames_cap(max_bits, f.cfg.cadu_size), 0, false);
    }
    const std::vector<uint16_t> cols_h = c2_rows();
    std::vector<int> ptr;
    std::vector<uint16_t> rows;
    level_schedule(cols_h, c.ldpc_iterations, ptr, rows);
    nlevels = (int)ptr.size() - 1;
    cols.alloc(cols_h.size());
    level_ptr.alloc(ptr.size());
    level_rows.alloc(std::max<size_t>(rows.size(), 1));
    unsigned char pnb[255];
    ccsds_pn_bits(pnb);
    pn.alloc(256);
    B200_CUDA(cudaMemcpyAsync(cols.p, cols_h.data(), cols_h.size() * sizeof(uint16_t), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaMemcpyAsync(level_ptr.p, ptr.data(), ptr.size() * sizeof(int), cudaMemcpyHostToDevice, f.stream));
    if (!rows.empty())
        B200_CUDA(cudaMemcpyAsync(level_rows.p, rows.data(), rows.size() * sizeof(uint16_t), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaMemcpyAsync(pn.p, pnb, 255, cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream)); // (the host vectors above die here)
}

std::unique_ptr<Decoder> ldpc_decoder(Fec &f) { return std::make_unique<Ldpc>(f); }

void Ldpc::reset(Fec &f)
{
    if (internal) {
        defr.start(f, 64);
        B200_CUDA(cudaStreamSynchronize(f.stream));
    }
    Correlated::reset(f);
    corr = 0;
}

// The module loop over every frame the FIFO completes: correlation at every position, the frame walk, then gather, decode and repack of
// all its frames at once (internal_stream: their info bits through the bit FIFO and the deframer).
void Ldpc::process(Fec &f)
{
    if (!begin(f, LDPC_F))
        return;
    if (internal)
        defr.compact(f);
    cudaStream_t stream = f.stream;
    const long have = f.soft_have, npos = have - (LDPC_ASM - 1);
    B200_CUDA(cudaEventRecord(ev[0], stream));
    k_ldpc_corr<<<(unsigned)((npos + 255) / 256), 256, 0, stream>>>(f.softbuf.p, npos, sw, nsync, score.p, bsync.p, bval.p, bidx.p);
    B200_CUDA(cudaEventRecord(ev[1], stream));
    const CorrWindow win{score.p, bsync.p, bval.p, bidx.p, LDPC_NPOS, constellation};
    k_frame_walk<<<1, WALK_WARPS * 32, 0, stream>>>(win, have, LDPC_F, frames.p, (int)max_frames, walk.p);
    B200_CUDA(cudaEventRecord(ev[2], stream));
    f.launches += 2;
    const int nf = walked(stream);
    if (nf > 0) {
        B200_REQUIRE(internal || (size_t)(f.out_frames + nf) * LDPC_CADU <= f.frames_out.n, B200_ESTATE,
                     "%ld frames not pulled yet: pull the frames between pushes", f.out_frames);
        k_ldpc_gather<<<nf, 256, 0, stream>>>(f.softbuf.p, frames.p, constellation == B200_OQPSK, derandomize ? pn.p : nullptr, vn.p);
        B200_CUDA(cudaEventRecord(ev[3], stream));
        const int smem = ((LDPC_VN * 2 + 15) & ~15) + LDPC_ROWS * (int)sizeof(LdpcRowMsg);
        uint8_t *cadu = internal ? cadu_tmp.p : f.frames_out.p + f.out_frames * LDPC_CADU;
        k_ldpc_decode<<<nf, LDPC_DEC_THREADS, smem, stream>>>(vn.p, cols.p, level_ptr.p, level_rows.p, nlevels, frames.p, cadu);
        f.launches += 2;
        B200_CUDA(cudaMemcpyAsync(h_frames.p, frames.p, sizeof(WalkFrame) * nf, cudaMemcpyDeviceToHost, stream));
        if (internal) { // :233-242: deframer->work(first 7136 decoded bits) of every codeword, in stream order
            const long new_bits = (long)nf * LDPC_INFO_BITS;
            const long words = (new_bits + 63) / 32;
            k_ldpc_append<<<(unsigned)std::min<long>((words + 255) / 256, 132 * 8), 256, 0, stream>>>(cadu, nf, defr.fifo.p, defr.fifo_bits);
            f.launches++;
            f.last_bits0 = defr.fifo_bits;
            f.last_nbits = new_bits;
            defr.deframe(f, fs, new_bits); // (synchronises the stream)
        }
        B200_CUDA(cudaEventRecord(ev[4], stream));
    }
    f.keep_soft_tail(h_walk.p->next);
    B200_CUDA(cudaEventRecord(ev[5], stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&t_ms[0], ev[0], ev[1]);
    cudaEventElapsedTime(&t_ms[1], ev[1], ev[2]);
    if (nf > 0) {
        cudaEventElapsedTime(&t_ms[2], ev[2], ev[3]);
        cudaEventElapsedTime(&t_ms[3], ev[3], ev[4]);
    }
    cudaEventElapsedTime(&t_ms[4], ev[0], ev[5]);
    f.t_vit = t_ms[4];
    finish(nf, f.soft_have);
    if (nf > 0)
        corr = h_frames.p[nf - 1].corr;
    if (!internal) { // (internal_stream: the frame stage counted the inner frames)
        f.out_frames += nf;
        f.total_frames += nf;
    }
    f.total_chunks += nf;
    f.total_bits += (long)nf * LDPC_CW;
}

void Ldpc::stats(b200_fec_stats *o)
{
    Correlated::stats(o);
    o->ldpc_corr = corr;
    o->deframer_state = defr.state_now;
}

long Ldpc::records(b200_ldpc_frame *out, long cap) const
{
    B200_REQUIRE(last_nf <= cap, B200_ESTATE, "output buffer too small: need %ld records", last_nf);
    for (long k = 0; k < last_nf; k++) {
        const WalkFrame &r = h_frames.p[k];
        out[k] = b200_ldpc_frame{(long)r.off, r.pos, r.cor, r.phase, r.swap, r.corr};
    }
    return last_nf;
}

void Ldpc::timing(float *ms, int n) const
{
    for (int k = 0; k < n && k < 5; k++)
        ms[k] = t_ms[k];
}

} // namespace b200

using namespace b200;

extern "C" {
int b200_fec_debug_ldpc_frames(b200_fec *h, b200_ldpc_frame *out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        *n_out = h->f->decoder_as<Ldpc>("not an LDPC decoder").records(out, cap);
    });
}
int b200_fec_ldpc_timing(b200_fec *h, float *ms_out, int n)
{
    return guarded([&] {
        B200_REQUIRE(h && ms_out, B200_EINVAL, "NULL argument");
        h->f->decoder_as<Ldpc>("not an LDPC decoder (kind B200_FEC_LDPC)").timing(ms_out, n);
    });
}
}
