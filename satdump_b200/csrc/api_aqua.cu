// Host driver of aqua_db_decoder (B200_FEC_AQUA_DB) inside the decoder object: AquaDBDecoderModule::process
// (plugins/eos_support/aqua/module_aqua_db_decoder.cpp:27-83) over the soft FIFO of Fec. Every push: the NRZ-M-decoded, interleaved bit
// stream of all its complete symbols (k_aqua_bits), then the deframer and frame stage the convolutional decoders use (k_deframe with the
// SYNCED state 10, k_frames with the derandomiser from byte 4, RS I=4 dual basis, every frame written).
#include "fec_host.h"
#include <algorithm>

namespace b200
{

// The soft FIFO starts with the previous push's last symbol (at a stream's start, the symbol (0, 0): both rails' NRZMDiff::lastBit = 0).
constexpr int AQUA_LEAD = 2;

// Soft pairs (I, Q) -> decoded bits. The module's interleaved hard bits are h(2s) = Q_s > 0 (rail A, demod >> 1) and h(2s + 1) = I_s > 0
// (rail B, demod & 1), that is h(k) = soft[k ^ 1] > 0; each rail's NRZMDiff::decode_bits XORs a bit with the same rail's bit one symbol
// earlier, so decoded bit j = h(j + 2) ^ h(j), with symbol 0 of `soft` the carried one. One warp writes one word of the MSB-first bit
// FIFO, which the stream enters at bit fifo_bits0 (the bits in front of it in the first word are kept).
__global__ void __launch_bounds__(256) k_aqua_bits(const int8_t *__restrict__ soft, long nbits, uint32_t *__restrict__ fifo, long fifo_bits0)
{
    const int lane = threadIdx.x & 31;
    const long w0 = fifo_bits0 >> 5, w1 = (fifo_bits0 + nbits + 31) >> 5;
    const long nwarps = (long)gridDim.x * (blockDim.x >> 5);
    for (long w = w0 + ((long)blockIdx.x * blockDim.x + threadIdx.x) / 32; w < w1; w += nwarps) {
        const long j = (w << 5) - fifo_bits0 + lane;
        const bool in = j >= 0 && j < nbits;
        const bool bit = in && ((soft[(j + 2) ^ 1] > 0) != (soft[j ^ 1] > 0));
        const uint32_t v = __brev(__ballot_sync(0xffffffffu, bit)), mask = __brev(__ballot_sync(0xffffffffu, in));
        if (lane == 0)
            fifo[w] = mask == 0xffffffffu ? v : ((fifo[w] & ~mask) | v);
    }
}

struct Aqua : Framed
{
    explicit Aqua(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
};

Aqua::Aqua(Fec &f)
{
    b200_fec_cfg &c = f.cfg;
    B200_REQUIRE(c.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for aqua_db_decoder");
    // BPSK_CCSDS_Deframer(8192, 0x1ACFFC1D) with STATE_SYNCED = 10 (:20-21), derand_ccsds(&cadu[4], 1020), decode_interlaved(&cadu[4], true, 4)
    c.cadu_size = 8192;
    c.asm_sync = 0x1ACFFC1D;
    c.nrzm = 0;
    c.derandomize = 1;
    c.derand_after_rs = 0;
    c.derand_start = 4;
    c.rs_i = 4;
    c.rs_dualbasis = 1;
    c.rs_type = 0;
    c.rs_fill_bytes = -1;
    c.rs_usecheck = 0;
    f.st_synced = 10;
    f.cadu_bytes = 1024;
    f.geom.chunk = 65536; // the module's read size (BUFFER_SIZE): what a stream reader of the decoder hands over at a time
    check_device(c.device);
    DeviceGuard g(c.device);
    f.framed_storage(2 * AQUA_LEAD, 0);
    f.deframer_storage(c.max_soft + 2 * AQUA_LEAD); // one bit per soft byte
    reset(f);
}

std::unique_ptr<Framed> aqua_decoder(Fec &f) { return std::make_unique<Aqua>(f); }

void Aqua::reset(Fec &f)
{
    f.start_stream(64); // the bit FIFO and the deframer
    Framed::reset(f);
    B200_CUDA(cudaMemsetAsync(f.softbuf.p, 0, AQUA_LEAD, f.stream));
    f.soft_have = AQUA_LEAD;
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

void Aqua::process(Fec &f)
{
    if (!begin(f, 2 * AQUA_LEAD)) // (no complete symbol behind the carried one)
        return;
    cudaStream_t stream = f.stream;
    f.compact_fifo(false);
    const long nbits = (f.soft_have / 2 - 1) * 2;
    B200_REQUIRE(((f.fifo_bits + nbits + 64) >> 5) + 2 < (long)f.fifo.n, B200_ESTATE, "internal: bit FIFO too small");
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    const long words = (f.fifo_bits + nbits + 31) / 32 - f.fifo_bits / 32;
    k_aqua_bits<<<(unsigned)std::min<long>((words + 7) / 8, 132 * 32), 256, 0, stream>>>(f.softbuf.p, nbits, f.fifo.p, f.fifo_bits);
    f.launches++;
    f.last_bits0 = f.fifo_bits;
    f.last_nbits = nbits;
    f.deframe_and_rs(nbits); // (synchronises the stream)
    f.keep_soft_tail(nbits); // the last symbol, the next push's predecessor, and an odd byte
    B200_CUDA(cudaEventRecord(f.ev[1], stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&f.t_vit, f.ev[0], f.ev[1]);
    f.t_vit -= f.t_frames;
    tail_seen = f.soft_have;
    f.total_bits += nbits;
}

} // namespace b200
