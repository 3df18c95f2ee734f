// C ABI of the CADU -> CCSDS space packet demultiplexer (include/b200dsp.h: b200_demux_*). Kernels in demux.cuh.
#define B200_DEFINE_KERNELS
#include "demux.cuh"
#include "host_common.h"
#include <algorithm>
#include <vector>

namespace b200
{

struct Demux
{
    b200_demux_cfg cfg;
    DmxGeom G;
    cudaStream_t stream = nullptr;
    long max_frames = 0, cap_recs = 0, cap_bytes = 0, frame0 = 0;
    int carry_cap = 1 << 17; // bytes of a packet under construction carried between pushes (a packet holds at most 65 550)
    int parity = 0;
    DevBuf<uint8_t> frames, fxa, fxb, carry[2], out;
    DevBuf<FrameSum> sums;
    DevBuf<int> cnt, tailseg, flags, sizes;
    DevBuf<unsigned long long> redo_mask;
    DevBuf<long> base, offs;
    DevBuf<WalkPkt> wp;
    DevBuf<DmxSeg> segs;
    DevBuf<PktRec> recs;
    DevBuf<DmxOut> orec;
    DevBuf<DmxCarry> st[2];
    PinnedBuf<long> h_counts; // packets, bytes
    PinnedBuf<int> h_flags;
    PinnedBuf<unsigned long long> h_redo;
    long redone_channels = 0; // channels walked again by one warp because a guess at a window boundary was wrong (so far)
    long last_packets = 0, last_bytes = 0, total_packets = 0, total_frames = 0, launches = 0;

    explicit Demux(const b200_demux_cfg &c) : cfg(c)
    {
        B200_REQUIRE(c.cadu_size >= 16 && c.cadu_size <= 65536, B200_EINVAL, "cadu_size out of range");
        B200_REQUIRE(c.mpdu_data_size >= 7 && c.mpdu_data_size < 2047, B200_EINVAL, "mpdu_data_size must be in [7, 2046]");
        B200_REQUIRE(c.insert_zone_size >= 0, B200_EINVAL, "insert_zone_size must not be negative");
        G.stride = c.cadu_size;
        G.data_off = 12 + (c.has_insert_zone ? c.insert_zone_size : 0); // mpdu.cpp:11-12
        G.M = c.mpdu_data_size;
        G.sec_ext = c.secondary_header_extends != 0;
        B200_REQUIRE(G.data_off + G.M <= c.cadu_size, B200_EINVAL, "M-PDU data zone (%d bytes at offset %d) does not fit a %d-byte CADU", G.M, G.data_off, c.cadu_size);
        B200_REQUIRE(c.max_frames >= 1, B200_EINVAL, "max_frames must be positive");
        max_frames = c.max_frames;
        check_device(c.device);
        DeviceGuard g(c.device);
        B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        cap_recs = c.max_packets > 0 ? c.max_packets : max_frames * 8 + 1024;
        cap_bytes = max_frames * (2L * G.M) + cap_recs * 6 + 64L * carry_cap;
        frames.alloc((size_t)max_frames * G.stride);
        sums.alloc(max_frames);
        fxa.alloc(max_frames);
        fxb.alloc(max_frames);
        cnt.alloc(max_frames);
        base.alloc(max_frames + 1);
        tailseg.alloc(128);
        flags.alloc(1);
        redo_mask.alloc(1);
        wp.alloc(2 * max_frames);       // two walk-packet slots per frame
        segs.alloc(3 * max_frames + 64); // three segment slots per frame + one carry segment per channel
        recs.alloc(cap_recs);
        orec.alloc(cap_recs);
        sizes.alloc(cap_recs);
        offs.alloc(cap_recs + 1);
        out.alloc(cap_bytes);
        for (int i = 0; i < 2; i++) {
            carry[i].alloc((size_t)64 * carry_cap);
            st[i].alloc(64);
            st[i].zero(stream);
        }
        h_counts.alloc(2);
        h_flags.alloc(1);
        h_redo.alloc(1);
        B200_CUDA(cudaStreamSynchronize(stream));
    }
    ~Demux()
    {
        DeviceGuard g(cfg.device);
        if (stream) {
            cudaStreamSynchronize(stream);
            cudaStreamDestroy(stream);
        }
    }
    void reset()
    {
        DeviceGuard g(cfg.device);
        for (int i = 0; i < 2; i++)
            st[i].zero(stream);
        B200_CUDA(cudaStreamSynchronize(stream));
        frame0 = 0;
        last_packets = last_bytes = 0;
    }
    void process(const uint8_t *d_frames, long n)
    {
        B200_REQUIRE(n >= 1 && n <= max_frames, B200_ESTATE, "%ld frames outside [1, max_frames %ld]", n, max_frames);
        DeviceGuard g(cfg.device);
        const int cur = parity, nxt = parity ^ 1;
        B200_CUDA(cudaMemsetAsync(fxa.p, 0, n, stream));
        B200_CUDA(cudaMemsetAsync(fxb.p, 0, n, stream));
        B200_CUDA(cudaMemsetAsync(flags.p, 0, sizeof(int), stream));
        B200_CUDA(cudaMemsetAsync(redo_mask.p, 0, sizeof(unsigned long long), stream));
        const unsigned fb = (unsigned)((n + 255) / 256);
        k_dmx_frames<false><<<fb, 256, 0, stream>>>(d_frames, n, frame0, G, cfg.vcid_mask, sums.p, nullptr, nullptr, nullptr, nullptr, 0, flags.p);
        // the walk: DMX_K guessing warps per channel, then one warp for every channel whose guess at a window boundary was wrong
        k_dmx_walk<<<dim3(DMX_K, 64), 32, 0, stream>>>(sums.p, n, frame0, G, 0, redo_mask.p, d_frames, st[cur].p, st[nxt].p, fxa.p, fxb.p, wp.p, segs.p, tailseg.p);
        k_dmx_walk<<<dim3(1, 64), 32, 0, stream>>>(sums.p, n, frame0, G, 1, redo_mask.p, d_frames, st[cur].p, st[nxt].p, fxa.p, fxb.p, wp.p, segs.p, tailseg.p);
        k_dmx_cnt<<<fb, 256, 0, stream>>>(sums.p, fxa.p, n, cnt.p);
        k_dmx_scan<<<1, 1024, 0, stream>>>(cnt.p, n, nullptr, base.p);
        k_dmx_frames<true><<<fb, 256, 0, stream>>>(d_frames, n, frame0, G, cfg.vcid_mask, nullptr, base.p, fxa.p, fxb.p, recs.p, cap_recs, flags.p);
        k_dmx_place<<<fb, 256, 0, stream>>>(wp.p, sums.p, fxa.p, fxb.p, n, base.p, recs.p, cap_recs, flags.p);
        B200_CUDA(cudaMemcpyAsync(h_redo.p, redo_mask.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaMemcpyAsync(&h_counts.p[0], base.p + n, sizeof(long), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaMemcpyAsync(h_flags.p, flags.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        B200_REQUIRE(!(*h_flags.p & 1) && h_counts.p[0] <= cap_recs, B200_ESTATE, "packet table too small: %ld packets in this batch, room for %ld (max_packets)",
                     h_counts.p[0], cap_recs);
        const long P = h_counts.p[0];
        k_dmx_sizes<<<(unsigned)std::min<long>(1024, (P + 255) / 256 + 1), 256, 0, stream>>>(recs.p, base.p + n, sizes.p);
        k_dmx_scan<<<1, 1024, 0, stream>>>(sizes.p, P, nullptr, offs.p);
        k_dmx_copy<<<(unsigned)std::min<long>(132 * 16, (P + 7) / 8 + 1), 256, 0, stream>>>(recs.p, base.p + n, offs.p, segs.p, d_frames, G, carry[cur].p, carry_cap, out.p,
                                                                                             cap_bytes, orec.p, flags.p);
        k_dmx_carry<<<64, 256, 0, stream>>>(tailseg.p, segs.p, d_frames, G, carry[cur].p, carry[nxt].p, carry_cap, flags.p);
        B200_CUDA(cudaMemcpyAsync(&h_counts.p[1], offs.p + P, sizeof(long), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaMemcpyAsync(h_flags.p, flags.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        B200_CUDA(cudaGetLastError());
        launches += 12;
        if (*h_redo.p)
            redone_channels += __builtin_popcountll(*h_redo.p);
        B200_REQUIRE(!(*h_flags.p & 2), B200_ESTATE, "internal: packet byte buffer too small");
        B200_REQUIRE(!(*h_flags.p & 4), B200_EUNSUPPORTED, "a packet under construction grew beyond %d bytes (inconsistent frames)", carry_cap);
        parity = nxt;
        frame0 += n;
        last_packets = P;
        last_bytes = h_counts.p[1];
        total_packets += P;
        total_frames += n;
    }
};

} // namespace b200

using namespace b200;
struct b200_demux_s
{
    Demux *d;
};

extern "C" {
b200_demuxer *b200_demux_create(const b200_demux_cfg *cfg)
{
    b200_demuxer *h = nullptr;
    int rc = guarded([&] {
        B200_REQUIRE(cfg, B200_EINVAL, "NULL cfg");
        h = reinterpret_cast<b200_demuxer *>(new b200_demux_s{new Demux(*cfg)});
    });
    return rc == B200_OK ? h : nullptr;
}
void b200_demux_destroy(b200_demuxer *h)
{
    if (!h)
        return;
    b200_demux_s *s = reinterpret_cast<b200_demux_s *>(h);
    delete s->d;
    delete s;
}
int b200_demux_push_frames(b200_demuxer *h, const uint8_t *host_cadus, long nframes)
{
    return guarded([&] {
        B200_REQUIRE(h && host_cadus, B200_EINVAL, "NULL argument");
        Demux &d = *reinterpret_cast<b200_demux_s *>(h)->d;
        B200_REQUIRE(nframes >= 1 && nframes <= d.max_frames, B200_ESTATE, "%ld frames outside [1, max_frames %ld]", nframes, d.max_frames);
        DeviceGuard g(d.cfg.device);
        B200_CUDA(cudaMemcpyAsync(d.frames.p, host_cadus, (size_t)nframes * d.G.stride, cudaMemcpyHostToDevice, d.stream));
        d.process(d.frames.p, nframes);
    });
}
int b200_demux_push_frames_device(b200_demuxer *h, const uint8_t *dev_cadus, long nframes)
{
    return guarded([&] {
        B200_REQUIRE(h && dev_cadus, B200_EINVAL, "NULL argument");
        reinterpret_cast<b200_demux_s *>(h)->d->process(dev_cadus, nframes);
    });
}
int b200_demux_pull(b200_demuxer *h, uint8_t *bytes, long cap_bytes, long *nbytes, b200_packet *packets, long cap_packets, long *npackets)
{
    return guarded([&] {
        B200_REQUIRE(h && nbytes && npackets, B200_EINVAL, "NULL argument");
        Demux &d = *reinterpret_cast<b200_demux_s *>(h)->d;
        B200_REQUIRE(d.last_bytes <= cap_bytes && d.last_packets <= cap_packets, B200_ESTATE, "output buffers too small: need %ld bytes, %ld packets", d.last_bytes,
                     d.last_packets);
        DeviceGuard g(d.cfg.device);
        static_assert(sizeof(b200_packet) == sizeof(DmxOut), "b200_packet layout");
        if (d.last_bytes)
            B200_CUDA(cudaMemcpyAsync(bytes, d.out.p, d.last_bytes, cudaMemcpyDeviceToHost, d.stream));
        if (d.last_packets)
            B200_CUDA(cudaMemcpyAsync(packets, d.orec.p, d.last_packets * sizeof(DmxOut), cudaMemcpyDeviceToHost, d.stream));
        B200_CUDA(cudaStreamSynchronize(d.stream));
        *nbytes = d.last_bytes;
        *npackets = d.last_packets;
        d.last_bytes = d.last_packets = 0;
    });
}
int b200_demux_reset(b200_demuxer *h)
{
    return guarded([&] {
        B200_REQUIRE(h, B200_EINVAL, "NULL handle");
        reinterpret_cast<b200_demux_s *>(h)->d->reset();
    });
}
int b200_demux_get_stats(b200_demuxer *h, b200_demux_stats *out)
{
    return guarded([&] {
        B200_REQUIRE(h && out, B200_EINVAL, "NULL argument");
        Demux &d = *reinterpret_cast<b200_demux_s *>(h)->d;
        out->frames_in = d.total_frames;
        out->packets_out = d.total_packets;
        out->kernel_launches = d.launches;
        out->redone_channels = d.redone_channels;
    });
}
}
