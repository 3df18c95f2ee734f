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

struct Turbo
{
    TurboGeom G{};
    TurboCode upper{}, lower{};
    int base = 0, iters = 0, batch = 0;
    double two_nv = 0, ln_half = 0;
    long tail_seen = -1; // FIFO bytes left by the last pass (a second process() without new bytes changes nothing)
    long max_frames = 0;
    DevBuf<float> score, bval, table, recv;
    DevBuf<int> bidx, perm;
    DevBuf<unsigned char> bsync, pn, bits;
    DevBuf<double> msg, bwd, fwd;
    DevBuf<LdpcFrameRec> frames;
    DevBuf<LdpcWalkOut> walk;
    DevBuf<uint8_t> cadu_tmp;
    DevBuf<unsigned long long> ties;
    LdpcWalkOut *h_walk = nullptr;
    LdpcFrameRec *h_frames = nullptr;
    unsigned long long *h_ties = nullptr;
    long last_nf = 0, last_b0 = 0; // frames of the last push; the first one of its last decoding batch
    long base_off = 0, resyncs = 0, crc_ok = 0, crc_fail = 0, near_ties = 0;
    int lock = 0;
    float cor = 0.f;
    cudaEvent_t ev[7]{};
    float t_ms[6]{}; // last push: correlation, walk, gather, BCJR, pack + CRC + compaction, the whole push
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
void Fec::turbo_init()
{
    const b200_fec_cfg &c = cfg;
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
    turbo = new Turbo();
    Turbo &T = *turbo;
    TurboGeom &G = T.G;
    T.base = c.turbo_base;
    T.iters = c.turbo_iters;
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
        T.upper = make_code({"10011", "11011", "10101", "11111"});
        T.lower = make_code({"11011", "11111"});
    } else {
        T.upper = c.turbo_rate == 4 ? make_code({"10011", "10101", "11111"}) : make_code({"10011", "11011"});
        T.lower = make_code({"11011"});
    }
    const float sigma = 0.707f; // CCSDSTurbo::d_sigma; turbo_decode gets d_sigma * d_sigma, a float product widened to double
    const float var = sigma * sigma;
    T.two_nv = 2 * (double)var;
    T.ln_half = std::log(0.5);
    geom.chunk = G.F;
    cadu_bytes = c.turbo_base + 4;
    cfg.cadu_size = cadu_bytes * 8;
    check_device(c.device);
    DeviceGuard g(c.device);
    B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    for (cudaEvent_t *e : {&ev[0], &ev[1], &evm[0], &evm[1], &evf[0], &evf[1]}) // (the destructor destroys all six)
        B200_CUDA(cudaEventCreate(e));
    for (auto &e : T.ev)
        B200_CUDA(cudaEventCreate(&e));
    const long fifo = c.max_soft + 2L * G.F;
    softbuf.alloc((size_t)fifo);
    dec.alloc((size_t)(2 * G.F) / sizeof(uint2) + 16); // scratch of keep_soft_tail
    T.score.alloc((size_t)fifo);
    T.bsync.alloc((size_t)fifo);
    T.bval.alloc((size_t)fifo / 32 + 2);
    T.bidx.alloc((size_t)fifo / 32 + 2);
    T.max_frames = fifo / G.F + 2;
    T.batch = (int)std::min<long>(T.max_frames, TURBO_BATCH);
    T.frames.alloc((size_t)T.max_frames);
    T.walk.alloc(1);
    T.recv.alloc((size_t)T.batch * G.recv_stride);
    T.msg.alloc((size_t)T.batch * 2 * G.K);
    T.bwd.alloc((size_t)T.batch * G.N * TURBO_STATES);
    T.fwd.alloc((size_t)T.batch * G.N * TURBO_STATES);
    T.bits.alloc((size_t)T.batch * G.K);
    T.cadu_tmp.alloc((size_t)T.max_frames * cadu_bytes);
    T.ties.alloc(1);
    max_frames_push = T.max_frames;
    frames_out.alloc((size_t)(2 * T.max_frames + 4) * cadu_bytes);
    const std::vector<int> pi = interleaver(c.turbo_base);
    T.perm.alloc(pi.size());
    const char *hex = asm_hex(c.turbo_rate);
    std::vector<float> table(G.asm_bits);
    for (int i = 0; i < G.asm_bits; i++) {
        const char h = hex[i / 4];
        const int nib = h <= '9' ? h - '0' : h - 'A' + 10;
        table[i] = (nib >> (3 - i % 4)) & 1 ? 1.0f : -1.0f;
    }
    T.table.alloc(table.size());
    unsigned char pnb[255];
    ccsds_pn_bits(pnb);
    T.pn.alloc(256);
    B200_CUDA(cudaMemcpyAsync(T.perm.p, pi.data(), pi.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMemcpyAsync(T.table.p, table.data(), table.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMemcpyAsync(T.pn.p, pnb, 255, cudaMemcpyHostToDevice, stream));
    T.ties.zero(stream);
    B200_CUDA(cudaFuncSetAttribute(k_turbo_pack, cudaFuncAttributeMaxDynamicSharedMemorySize, T.base));
    B200_CUDA(cudaMallocHost((void **)&T.h_walk, sizeof(LdpcWalkOut)));
    B200_CUDA(cudaMallocHost((void **)&T.h_frames, sizeof(LdpcFrameRec) * T.max_frames));
    B200_CUDA(cudaMallocHost((void **)&T.h_ties, sizeof(unsigned long long)));
    B200_CUDA(cudaStreamSynchronize(stream)); // (the host vectors above die here)
}

void Fec::turbo_free()
{
    if (!turbo)
        return;
    for (auto &e : turbo->ev)
        if (e)
            cudaEventDestroy(e);
    for (void *p : {(void *)turbo->h_walk, (void *)turbo->h_frames, (void *)turbo->h_ties})
        if (p)
            cudaFreeHost(p);
    delete turbo;
    turbo = nullptr;
}

void Fec::turbo_reset()
{
    soft_have = 0;
    out_frames = 0;
    Turbo &T = *turbo;
    T.tail_seen = -1;
    T.base_off = 0;
    T.last_nf = 0;
    T.lock = 0;
    T.cor = 0.f;
    T.near_ties = 0;
    T.ties.zero(stream);
    B200_CUDA(cudaStreamSynchronize(stream));
}

// The module loop over every frame the FIFO completes: correlation at every position and the frame walk, then, batch by batch, gather,
// turbo_iters x (upper BCJR, lower BCJR) and the CRC; the frames that pass are compacted into frames_out. The bytes behind the walk's
// next window stay in the FIFO; a call that finds no new bytes behind them has nothing to do.
void Fec::turbo_process()
{
    Turbo &T = *turbo;
    const TurboGeom &G = T.G;
    if (soft_have == T.tail_seen)
        return;
    T.last_nf = 0;
    for (float &t : T.t_ms)
        t = 0;
    if (soft_have < G.F) {
        T.tail_seen = soft_have;
        return;
    }
    const long have = soft_have, npos = have - (G.asm_bits - 1);
    B200_CUDA(cudaEventRecord(T.ev[0], stream));
    switch (G.asm_bits) {
    case 64: launch_corr<64>(softbuf.p, npos, T, stream); break;
    case 96: launch_corr<96>(softbuf.p, npos, T, stream); break;
    case 128: launch_corr<128>(softbuf.p, npos, T, stream); break;
    default: launch_corr<192>(softbuf.p, npos, T, stream); break;
    }
    B200_CUDA(cudaEventRecord(T.ev[1], stream));
    frame_walk(T.score.p, T.bsync.p, T.bval.p, T.bidx.p, have, G.F, G.F - G.asm_bits, WALK_SWAP_ONLY, T.frames.p, (int)T.max_frames, T.walk.p,
               stream);
    B200_CUDA(cudaEventRecord(T.ev[2], stream));
    launches += 2;
    B200_CUDA(cudaMemcpyAsync(T.h_walk, T.walk.p, sizeof(LdpcWalkOut), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    const int nf = T.h_walk->nf;
    float t_gather = 0, t_bcjr = 0;
    if (nf > 0) {
        B200_REQUIRE((size_t)(out_frames + nf) * cadu_bytes <= frames_out.n, B200_ESTATE, "%ld frames not pulled yet: pull the frames between pushes",
                     out_frames);
        for (int b0 = 0; b0 < nf; b0 += T.batch) {
            const int nb = std::min(T.batch, nf - b0);
            T.last_b0 = b0;
            B200_CUDA(cudaEventRecord(T.ev[3], stream));
            k_turbo_gather<<<nb, 256, 0, stream>>>(softbuf.p, T.frames.p + b0, G, T.pn.p, T.recv.p, T.msg.p, T.ln_half);
            B200_CUDA(cudaEventRecord(T.ev[4], stream));
            for (int it = 0; it < T.iters; it++) {
                half_iteration(T, nb, false, nullptr, stream);
                half_iteration(T, nb, true, it == T.iters - 1 ? T.bits.p : nullptr, stream);
            }
            B200_CUDA(cudaEventRecord(T.ev[5], stream));
            k_turbo_pack<<<nb, 256, T.base, stream>>>(T.bits.p, T.base, T.frames.p + b0, T.cadu_tmp.p + (size_t)b0 * cadu_bytes);
            launches += 2 + 4L * T.iters;
            B200_CUDA(cudaEventSynchronize(T.ev[5]));
            float a = 0, b = 0;
            cudaEventElapsedTime(&a, T.ev[3], T.ev[4]);
            cudaEventElapsedTime(&b, T.ev[4], T.ev[5]);
            t_gather += a;
            t_bcjr += b;
        }
        k_turbo_compact<<<nf, 256, 0, stream>>>(T.cadu_tmp.p, T.frames.p, cadu_bytes, frames_out.p + out_frames * cadu_bytes);
        launches++;
        B200_CUDA(cudaMemcpyAsync(T.h_frames, T.frames.p, sizeof(LdpcFrameRec) * nf, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaMemcpyAsync(T.h_ties, T.ties.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
    }
    B200_CUDA(cudaEventRecord(T.ev[6], stream));
    keep_soft_tail(T.h_walk->next);
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&T.t_ms[0], T.ev[0], T.ev[1]);
    cudaEventElapsedTime(&T.t_ms[1], T.ev[1], T.ev[2]);
    T.t_ms[2] = t_gather;
    T.t_ms[3] = t_bcjr;
    if (nf > 0) {
        float tail = 0, whole = 0;
        cudaEventElapsedTime(&tail, T.ev[5], T.ev[6]);
        cudaEventElapsedTime(&whole, T.ev[0], T.ev[6]);
        T.t_ms[4] = whole - T.t_ms[0] - T.t_ms[1] - t_gather - t_bcjr; // the pack launches of all batches, compaction and copies
        T.t_ms[5] = whole;
    } else
        T.t_ms[5] = T.t_ms[0] + T.t_ms[1];
    t_vit = T.t_ms[5];
    int ok = 0;
    for (int k = 0; k < nf; k++) {
        LdpcFrameRec &r = T.h_frames[k];
        r.off += T.base_off;
        T.resyncs += r.pos != 0;
        ok += r.corr != 0;
    }
    if (nf > 0) {
        const LdpcFrameRec &r = T.h_frames[nf - 1];
        T.lock = r.pos == 0;
        T.cor = r.cor;
        T.near_ties = (long)*T.h_ties;
    }
    T.crc_ok += ok;
    T.crc_fail += nf - ok;
    T.last_nf = nf;
    T.base_off += T.h_walk->next;
    T.tail_seen = soft_have;
    out_frames += ok;
    total_frames += ok;
    total_chunks += nf;
    total_bits += (long)ok * T.base * 8;
}

void Fec::turbo_stats(b200_fec_stats *o)
{
    o->correlator_lock = turbo->lock;
    o->correlator_corr = turbo->cor;
    o->ldpc_resyncs = turbo->resyncs;
    o->crc_ok = turbo->crc_ok;
    o->crc_fail = turbo->crc_fail;
    o->turbo_near_ties = turbo->near_ties;
}

long Fec::turbo_frames(b200_turbo_frame *out, long cap)
{
    B200_REQUIRE(turbo, B200_EINVAL, "not a turbo decoder");
    B200_REQUIRE(turbo->last_nf <= cap, B200_ESTATE, "output buffer too small: need %ld records", turbo->last_nf);
    for (long k = 0; k < turbo->last_nf; k++) {
        const LdpcFrameRec &r = turbo->h_frames[k];
        out[k] = b200_turbo_frame{(long)r.off, r.pos, r.cor, r.swap, r.corr};
    }
    return turbo->last_nf;
}

long Fec::turbo_llr(long frame, double *app0, double *app1, long cap)
{
    B200_REQUIRE(turbo, B200_EINVAL, "not a turbo decoder");
    Turbo &T = *turbo;
    const int K = T.G.K;
    B200_REQUIRE(frame >= T.last_b0 && frame < T.last_nf, B200_ESTATE, "frame %ld is not in the last decoding batch [%ld, %ld) of the last push",
                 frame, T.last_b0, T.last_nf);
    B200_REQUIRE(cap >= K, B200_ESTATE, "output buffer too small: need %d values", K);
    const double *m = T.msg.p + (size_t)(frame - T.last_b0) * 2 * K;
    B200_CUDA(cudaMemcpyAsync(app0, m, sizeof(double) * K, cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(app1, m + K, sizeof(double) * K, cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    return K;
}

void Fec::turbo_timing(float *ms, int n)
{
    for (int k = 0; k < n && k < 6; k++)
        ms[k] = turbo->t_ms[k];
}

} // namespace b200
