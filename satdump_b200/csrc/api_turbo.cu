// Host driver of ccsds_turbo_decoder (B200_FEC_TURBO) inside the decoder object: CCSDSTurboDecoderModule::process
// (src-core/pipeline/modules/ccsds/module_ccsds_turbo_decoder.cpp:137-235) over the soft FIFO of Fec, with CCSDSTurbo::decode
// (common/codings/turbo/ccsds_turbo.cpp:156-198) and turbo_decode (libs/deepspace-turbo/libturbocodes.c:137-201) on the device.
#include "fec_host.h"
#include "turbo.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

namespace b200
{

constexpr int TURBO_BATCH = 1024; // frames decoded at once: their BCJR metrics take 2 (K + 4) x 16 doubles each (2.3 MB at base 1115)

struct Turbo : Correlated
{
    TurboGeom G{};
    TurboCode upper{}, lower{};
    int base = 0, iters = 0, batch = 0;
    double two_nv = 0, ln_half = 0;
    DevBuf<float> table, recv;
    DevBuf<int> perm;
    DevBuf<unsigned char> pn, bits;
    DevBuf<double> msg, bwd, fwd;
    DevBuf<uint8_t> cadu_tmp;
    DevBuf<unsigned long long> ties;
    PinnedBuf<unsigned long long> h_ties;
    long last_b0 = 0; // the first frame of the last push's last decoding batch
    long crc_ok = 0, crc_fail = 0, near_ties = 0;
    Events<7> ev; // t_ms: correlation, walk, gather, BCJR, pack + CRC + compaction, the whole push

    explicit Turbo(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
    void stats(b200_fec_stats *o) override;
    long records(b200_turbo_frame *out, long cap) const; // of the last push
    long llr(cudaStream_t stream, long frame, double *app0, double *app1, long cap) const;
    void timing(float *ms, int n) const;
};

namespace
{
// The ASMs of the module's constructor (:38-117): 0x034776C7272895B0 (1/2), 0x25D5C0CE8990F6C9461BF79C (1/3),
// 0x034776C7272895B0FCB88938D8D76A4F (1/4), 0x25D5C0CE8990F6C9461BF79CDA2A3F31766F0936B9E40863 (1/6), MSB first
const char *asm_hex(int rate)
{
    switch (rate) {
    case 2: return "034776C7272895B0";
    case 3: return "25D5C0CE8990F6C9461BF79C";
    case 4: return "034776C7272895B0FCB88938D8D76A4F";
    default: return "25D5C0CE8990F6C9461BF79CDA2A3F31766F0936B9E40863";
    }
}

// The trellis of a recursive systematic component code with feedback "0011" and the given feed-forward polynomials (CCSDS 131.0-B,
// section 6): the new first register is input + the feedback taps of the state; output c = tap 0 x new first register + taps 1..4 x
// the state's registers (bit m-1-i of the state is register i). Predecessors in the order convcode_initialize files them: states
// ascending, input 0 before input 1 of each.
TurboCode make_code(const std::vector<const char *> &fwd)
{
    const char *bwd = "0011";
    TurboCode c{};
    auto reg = [](int st, int i) { return (st >> (TURBO_MEM - 1 - i)) & 1; };
    int filled[TURBO_STATES] = {};
    for (int st = 0; st < TURBO_STATES; st++)
        for (int u = 0; u < 2; u++) {
            int first = u;
            for (int i = 0; i < TURBO_MEM; i++)
                first ^= (bwd[i] - '0') & reg(st, i);
            const int ns = (st >> 1) | (first << (TURBO_MEM - 1));
            unsigned out = 0;
            for (size_t k = 0; k < fwd.size(); k++) {
                int o = (fwd[k][0] - '0') & first;
                for (int i = 0; i < TURBO_MEM; i++)
                    o ^= (fwd[k][i + 1] - '0') & reg(st, i);
                out |= (unsigned)o << k;
            }
            c.next[st][u] = (int8_t)ns;
            c.out[st][u] = (uint8_t)out;
            c.prev[ns][filled[ns]] = (int8_t)st;
            c.prev_u[ns][filled[ns]] = (int8_t)u;
            filled[ns]++;
        }
    return c;
}

// The CCSDS turbo interleaver (CCSDS 131.0-B section 6.3; the CCSDSTurbo constructor) for k = 8 base information bits
std::vector<int> interleaver(int base)
{
    const int p[8] = {31, 37, 43, 47, 53, 59, 61, 67}, k1 = 8, k2 = base, K = 8 * base;
    std::vector<int> pi(K);
    for (int s = 1; s <= K; s++) {
        const int m = (s - 1) % 2, i = (s - 1) / (2 * k2), j = (s - 1) / 2 - i * k2, t = (19 * i + 1) % (k1 / 2), q = t % 8 + 1;
        const int c = (p[q - 1] * j + 21 * m) % k2;
        pi[s - 1] = 2 * (t + c * (k1 / 2) + 1) - m - 1;
    }
    return pi;
}

template <int C>
void launch_rec(const Turbo &T, int nf, bool lower, const TurboCode &code, cudaStream_t st)
{
    const int warps = 2 * ((nf + 1) / 2), wpb = TURBO_REC_THREADS / 32;
    k_turbo_rec<C><<<(warps + wpb - 1) / wpb, TURBO_REC_THREADS, 0, st>>>(T.recv.p, lower ? T.G.cu * T.G.N : 0, T.msg.p, lower ? T.perm.p : nullptr,
                                                                       T.G, code, T.two_nv, T.ln_half, T.bwd.p, T.fwd.p, nf);
}
template <int C>
void launch_ext(const Turbo &T, int nf, bool lower, const TurboCode &code, unsigned char *bits, cudaStream_t st)
{
    const dim3 grid((T.G.N + TURBO_EXT_THREADS - 1) / TURBO_EXT_THREADS, nf);
    k_turbo_ext<C><<<grid, TURBO_EXT_THREADS, 0, st>>>(T.recv.p, lower ? T.G.cu * T.G.N : 0, T.msg.p, lower ? T.perm.p : nullptr, T.G, code,
                                                       T.two_nv, T.ln_half, T.bwd.p, T.fwd.p, bits, T.ties.p);
}
void half_iteration(const Turbo &T, int nf, bool lower, unsigned char *bits, cudaStream_t st)
{
    const TurboCode &code = lower ? T.lower : T.upper;
    switch (lower ? T.G.cl : T.G.cu) {
    case 1: launch_rec<1>(T, nf, lower, code, st); launch_ext<1>(T, nf, lower, code, bits, st); break;
    case 2: launch_rec<2>(T, nf, lower, code, st); launch_ext<2>(T, nf, lower, code, bits, st); break;
    case 3: launch_rec<3>(T, nf, lower, code, st); launch_ext<3>(T, nf, lower, code, bits, st); break;
    default: launch_rec<4>(T, nf, lower, code, st); launch_ext<4>(T, nf, lower, code, bits, st); break;
    }
}

template <int ASM>
void launch_corr(const int8_t *soft, long npos, Turbo &T, cudaStream_t st)
{
    k_turbo_corr<ASM><<<(unsigned)((npos + 255) / 256), 256, 0, st>>>(soft, npos, T.table.p, T.score.p, T.bsync.p, T.bval.p, T.bidx.p);
}
} // namespace

// The module's parameter checks (:20-36, :118-119), and the iteration count, refused by name before the device is touched
Turbo::Turbo(Fec &f)
{
    const b200_fec_cfg &c = f.cfg;
    B200_REQUIRE(c.turbo_rate != 0, B200_EINVAL, "Turbo Rate is required!");
    B200_REQUIRE(c.turbo_base != 0, B200_EINVAL, "Turbo Base is required!");
    B200_REQUIRE(c.turbo_base == 223 || c.turbo_base == 446 || c.turbo_base == 892 || c.turbo_base == 1115, B200_EINVAL,
                 "Turbo Base must be 223, 446, 892 or 1115!");
    B200_REQUIRE(c.turbo_rate == 2 || c.turbo_rate == 3 || c.turbo_rate == 4 || c.turbo_rate == 6, B200_EINVAL,
                 "Invalid Turbo Rate! (turbo_rate %d: 2, 3, 4, 6 = \"1/2\", \"1/3\", \"1/4\", \"1/6\")", c.turbo_rate);
    B200_REQUIRE(c.turbo_iters >= 1, B200_EINVAL,
                 "turbo_iters %d: at least 1 iteration is needed (with 0 the reference decodes nothing and dereferences NULL)", c.turbo_iters);
    B200_REQUIRE(c.turbo_iters <= 10000, B200_EINVAL, "turbo_iters out of range (1..10000)");
    B200_REQUIRE(c.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for the turbo decoder");
    base = c.turbo_base;
    iters = c.turbo_iters;
    G.K = 8 * c.turbo_base;
    G.N = G.K + TURBO_MEM;
    G.asm_bits = c.turbo_rate == 2 ? 64 : (c.turbo_rate == 3 ? 96 : (c.turbo_rate == 4 ? 128 : 192));
    G.cu = c.turbo_rate == 4 ? 3 : (c.turbo_rate == 6 ? 4 : 2);
    G.cl = c.turbo_rate == 6 ? 2 : 1;
    G.punct = c.turbo_rate == 2;
    G.cw = G.punct ? 2 * G.N : (G.cu + G.cl) * G.N; // 17848 / 26772 / 35696 / 53544 soft bytes at base 1115
    G.F = G.cw + G.asm_bits;
    G.recv_stride = (long)(G.cu + G.cl) * G.N;
    if (c.turbo_rate == 6) {
        upper = make_code({"10011", "11011", "10101", "11111"});
        lower = make_code({"11011", "11111"});
    } else {
        upper = c.turbo_rate == 4 ? make_code({"10011", "10101", "11111"}) : make_code({"10011", "11011"});
        lower = make_code({"11011"});
    }
    const float sigma = 0.707f; // CCSDSTurbo::d_sigma; turbo_decode gets d_sigma * d_sigma, a float product widened to double
    const float var = sigma * sigma;
    two_nv = 2 * (double)var;
    ln_half = std::log(0.5);
    f.chunk = G.F;
    f.cadu_bytes = c.turbo_base + 4;
    check_device(c.device);
    DeviceGuard g(c.device);
    const long fifo = c.max_soft + 2L * G.F;
    alloc(fifo, fifo / G.F + 2);
    f.open(G.F, max_frames);
    ev.create();
    batch = (int)std::min<long>(max_frames, TURBO_BATCH);
    recv.alloc((size_t)batch * G.recv_stride);
    msg.alloc((size_t)batch * 2 * G.K);
    bwd.alloc((size_t)batch * G.N * TURBO_STATES);
    fwd.alloc((size_t)batch * G.N * TURBO_STATES);
    bits.alloc((size_t)batch * G.K);
    cadu_tmp.alloc((size_t)max_frames * f.cadu_bytes);
    ties.alloc(1);
    h_ties.alloc(1);
    const std::vector<int> pi = interleaver(c.turbo_base);
    perm.alloc(pi.size());
    const char *hex = asm_hex(c.turbo_rate);
    std::vector<float> table_h(G.asm_bits);
    for (int i = 0; i < G.asm_bits; i++) {
        const char h = hex[i / 4];
        const int nib = h <= '9' ? h - '0' : h - 'A' + 10;
        table_h[i] = (nib >> (3 - i % 4)) & 1 ? 1.0f : -1.0f;
    }
    table.alloc(table_h.size());
    unsigned char pnb[255];
    ccsds_pn_bits(pnb);
    pn.alloc(256);
    B200_CUDA(cudaMemcpyAsync(perm.p, pi.data(), pi.size() * sizeof(int), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaMemcpyAsync(table.p, table_h.data(), table_h.size() * sizeof(float), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaMemcpyAsync(pn.p, pnb, 255, cudaMemcpyHostToDevice, f.stream));
    ties.zero(f.stream);
    B200_CUDA(cudaFuncSetAttribute(k_turbo_pack, cudaFuncAttributeMaxDynamicSharedMemorySize, base));
    B200_CUDA(cudaStreamSynchronize(f.stream)); // (the host vectors above die here)
}

std::unique_ptr<Decoder> turbo_decoder(Fec &f) { return std::make_unique<Turbo>(f); }

void Turbo::reset(Fec &f)
{
    Correlated::reset(f);
    near_ties = 0;
    ties.zero(f.stream);
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

// The module loop over every frame the FIFO completes: correlation at every position and the frame walk, then, batch by batch, gather,
// turbo_iters x (upper BCJR, lower BCJR) and the CRC; the frames that pass are compacted into frames_out.
void Turbo::process(Fec &f)
{
    if (!begin(f, G.F))
        return;
    cudaStream_t stream = f.stream;
    const long have = f.soft_have, npos = have - (G.asm_bits - 1);
    B200_CUDA(cudaEventRecord(ev[0], stream));
    switch (G.asm_bits) {
    case 64: launch_corr<64>(f.softbuf.p, npos, *this, stream); break;
    case 96: launch_corr<96>(f.softbuf.p, npos, *this, stream); break;
    case 128: launch_corr<128>(f.softbuf.p, npos, *this, stream); break;
    default: launch_corr<192>(f.softbuf.p, npos, *this, stream); break;
    }
    B200_CUDA(cudaEventRecord(ev[1], stream));
    const CorrWindow win{score.p, bsync.p, bval.p, bidx.p, G.F - G.asm_bits, WALK_SWAP_ONLY};
    k_frame_walk<<<1, WALK_WARPS * 32, 0, stream>>>(win, have, G.F, frames.p, (int)max_frames, walk.p);
    B200_CUDA(cudaEventRecord(ev[2], stream));
    f.launches += 2;
    const int nf = walked(stream);
    const int cadu_bytes = f.cadu_bytes;
    float t_gather = 0, t_bcjr = 0;
    if (nf > 0) {
        B200_REQUIRE((size_t)(f.out_frames + nf) * cadu_bytes <= f.frames_out.n, B200_ESTATE,
                     "%ld frames not pulled yet: pull the frames between pushes", f.out_frames);
        for (int b0 = 0; b0 < nf; b0 += batch) {
            const int nb = std::min(batch, nf - b0);
            last_b0 = b0;
            B200_CUDA(cudaEventRecord(ev[3], stream));
            k_turbo_gather<<<nb, 256, 0, stream>>>(f.softbuf.p, frames.p + b0, G, pn.p, recv.p, msg.p, ln_half);
            B200_CUDA(cudaEventRecord(ev[4], stream));
            for (int it = 0; it < iters; it++) {
                half_iteration(*this, nb, false, nullptr, stream);
                half_iteration(*this, nb, true, it == iters - 1 ? bits.p : nullptr, stream);
            }
            B200_CUDA(cudaEventRecord(ev[5], stream));
            k_turbo_pack<<<nb, 256, base, stream>>>(bits.p, base, frames.p + b0, cadu_tmp.p + (size_t)b0 * cadu_bytes);
            f.launches += 2 + 4L * iters;
            B200_CUDA(cudaEventSynchronize(ev[5]));
            float a = 0, b = 0;
            cudaEventElapsedTime(&a, ev[3], ev[4]);
            cudaEventElapsedTime(&b, ev[4], ev[5]);
            t_gather += a;
            t_bcjr += b;
        }
        k_turbo_compact<<<nf, 256, 0, stream>>>(cadu_tmp.p, frames.p, cadu_bytes, f.frames_out.p + f.out_frames * cadu_bytes);
        f.launches++;
        B200_CUDA(cudaMemcpyAsync(h_frames.p, frames.p, sizeof(WalkFrame) * nf, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaMemcpyAsync(h_ties.p, ties.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
    }
    B200_CUDA(cudaEventRecord(ev[6], stream));
    f.keep_soft_tail(h_walk.p->next);
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&t_ms[0], ev[0], ev[1]);
    cudaEventElapsedTime(&t_ms[1], ev[1], ev[2]);
    t_ms[2] = t_gather;
    t_ms[3] = t_bcjr;
    if (nf > 0) {
        float whole = 0;
        cudaEventElapsedTime(&whole, ev[0], ev[6]);
        t_ms[4] = whole - t_ms[0] - t_ms[1] - t_gather - t_bcjr; // the pack launches of all batches, compaction and copies
        t_ms[5] = whole;
    } else
        t_ms[5] = t_ms[0] + t_ms[1];
    f.t_vit = t_ms[5];
    finish(nf, f.soft_have);
    int ok = 0;
    for (int k = 0; k < nf; k++)
        ok += h_frames.p[k].corr != 0;
    if (nf > 0)
        near_ties = (long)*h_ties.p;
    crc_ok += ok;
    crc_fail += nf - ok;
    f.out_frames += ok;
    f.total_frames += ok;
    f.total_chunks += nf;
    f.total_bits += (long)ok * base * 8;
}

void Turbo::stats(b200_fec_stats *o)
{
    Correlated::stats(o);
    o->crc_ok = crc_ok;
    o->crc_fail = crc_fail;
    o->turbo_near_ties = near_ties;
}

long Turbo::records(b200_turbo_frame *out, long cap) const
{
    B200_REQUIRE(last_nf <= cap, B200_ESTATE, "output buffer too small: need %ld records", last_nf);
    for (long k = 0; k < last_nf; k++) {
        const WalkFrame &r = h_frames.p[k];
        out[k] = b200_turbo_frame{(long)r.off, r.pos, r.cor, r.swap, r.corr};
    }
    return last_nf;
}

long Turbo::llr(cudaStream_t stream, long frame, double *app0, double *app1, long cap) const
{
    const int K = G.K;
    B200_REQUIRE(frame >= last_b0 && frame < last_nf, B200_ESTATE, "frame %ld is not in the last decoding batch [%ld, %ld) of the last push",
                 frame, last_b0, last_nf);
    B200_REQUIRE(cap >= K, B200_ESTATE, "output buffer too small: need %d values", K);
    const double *m = msg.p + (size_t)(frame - last_b0) * 2 * K;
    B200_CUDA(cudaMemcpyAsync(app0, m, sizeof(double) * K, cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(app1, m + K, sizeof(double) * K, cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    return K;
}

void Turbo::timing(float *ms, int n) const
{
    for (int k = 0; k < n && k < 6; k++)
        ms[k] = t_ms[k];
}

} // namespace b200

using namespace b200;

extern "C" {
int b200_fec_debug_turbo_frames(b200_fec *h, b200_turbo_frame *out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        *n_out = h->f->decoder_as<Turbo>("not a turbo decoder").records(out, cap);
    });
}
int b200_fec_debug_turbo_llr(b200_fec *h, long frame, double *app0, double *app1, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && app0 && app1 && n_out, B200_EINVAL, "NULL argument");
        DeviceGuard g(h->f->cfg.device);
        *n_out = h->f->decoder_as<Turbo>("not a turbo decoder").llr(h->f->stream, frame, app0, app1, cap);
    });
}
int b200_fec_turbo_timing(b200_fec *h, float *ms_out, int n)
{
    return guarded([&] {
        B200_REQUIRE(h && ms_out, B200_EINVAL, "NULL argument");
        h->f->decoder_as<Turbo>("not a turbo decoder (kind B200_FEC_TURBO)").timing(ms_out, n);
    });
}
}
