// C ABI of the fused chain: demodulator + decoder of one stream on one GPU, the int8 soft stream handed over in HBM
// (the reference joins the two modules with a 1 MB host ring buffer: src-core/pipeline/pipeline_run.cpp:72-104).
#include "demod_host.h"
#include "fec_host.h"
#include <condition_variable>
#include <mutex>
#include <thread>

namespace b200
{
// Two modes.
//  * synchronous (default): push = demodulate, then decode, on the calling thread; the frames of a push can be pulled when it
//    returns.
//  * pipelined (b200_chain_set_pipelined): the decoder runs on a worker thread and its own CUDA stream, one batch behind the
//    demodulator - the two-module concurrency of the reference's Pipeline::run (pipeline_run.cpp:44-117: one thread per module
//    joined by a FIFO), here with the FIFO element being a whole batch of soft symbols in HBM. push(i) demodulates batch i while
//    the worker decodes batch i-1; the latency-bound loop kernels and the ALU-bound Viterbi kernel then share the SMs. Frames
//    appear one push later; b200_chain_sync() drains.
struct Chain
{
    Demod *d = nullptr;
    Fec *f = nullptr;
    float t_total = 0;
    cudaEvent_t e0 = nullptr, e1 = nullptr, span0 = nullptr, span1 = nullptr;

    bool pipelined = false;
    std::thread worker;
    std::mutex mu;
    std::condition_variable cv;
    bool busy = false, stop = false; // busy: a batch is queued or being decoded
    long job_bytes = 0;
    int job_buf = 0, cur = 0;
    bool job_reset = false, reset_pending = false; // a reset in pipelined mode reaches the decoder with the next batch
    DevBuf<int8_t> stage[2];          // soft symbols of the batch being demodulated / being decoded
    DevBuf<uint8_t> ready;            // frames of completed batches, swapped out of the decoder so pull never races it
    long ready_frames = 0;
    int err_code = 0;
    std::string err_msg;

    void wait_idle_locked(std::unique_lock<std::mutex> &lk)
    {
        cv.wait(lk, [&] { return !busy; });
        if (err_code) {
            const int c = err_code;
            const std::string m = err_msg;
            err_code = 0;
            throw ApiError(c, m.c_str());
        }
    }
    void sync()
    {
        if (!pipelined)
            return;
        std::unique_lock<std::mutex> lk(mu);
        wait_idle_locked(lk);
    }
    void run_worker()
    {
        for (;;) {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return stop || busy; });
            if (stop)
                return;
            const long nb = job_bytes;
            const int8_t *src = stage[job_buf].p;
            const bool rst = job_reset;
            lk.unlock();
            try {
                if (rst) {
                    stash_frames(); // the old stream's decoded frames stay pullable
                    f->reset();
                }
                f->push(src, nb, cudaMemcpyDeviceToDevice);
                f->process();
                DeviceGuard g(f->cfg.device);
                B200_CUDA(cudaEventRecord(e1, f->stream));
                B200_CUDA(cudaEventSynchronize(e1));
            } catch (const ApiError &e) {
                lk.lock();
                err_code = e.code;
                err_msg = e.what();
                lk.unlock();
            } catch (const std::exception &e) {
                lk.lock();
                err_code = B200_ECUDA;
                err_msg = e.what();
                lk.unlock();
            }
            lk.lock();
            if (ready_frames == 0 && f->out_frames > 0) { // hand the finished frames over
                std::swap(ready.p, f->frames_out.p);
                std::swap(ready.n, f->frames_out.n);
                ready_frames = f->out_frames;
                f->out_frames = 0;
            }
            busy = false;
            lk.unlock();
            cv.notify_all();
        }
    }
    // worker thread, decoder idle: move whatever the decoder holds behind the frames waiting in `ready`
    void stash_frames()
    {
        std::unique_lock<std::mutex> lk(mu);
        if (f->out_frames == 0)
            return;
        if (ready_frames == 0) {
            std::swap(ready.p, f->frames_out.p);
            std::swap(ready.n, f->frames_out.n);
        } else {
            DeviceGuard g(f->cfg.device);
            B200_REQUIRE((size_t)(ready_frames + f->out_frames) * f->cadu_bytes <= ready.n, B200_ESTATE,
                         "pipelined chain: too many decoded frames waiting to be pulled");
            B200_CUDA(cudaMemcpyAsync(ready.p + ready_frames * f->cadu_bytes, f->frames_out.p, f->out_frames * f->cadu_bytes, cudaMemcpyDeviceToDevice,
                                      f->stream));
            B200_CUDA(cudaStreamSynchronize(f->stream));
        }
        ready_frames += f->out_frames;
        f->out_frames = 0;
    }
    void set_pipelined(bool on)
    {
        if (on == pipelined)
            return;
        if (!on) {
            shutdown_worker();
            pipelined = false;
            return;
        }
        DeviceGuard g(d->cfg.device);
        const double omin = d->sps * (1.0 - d->cfg.clock_omega_limit) - 0.01;
        const size_t cap = (size_t)(d->max_work / omin + 1024) * d->bps; // max_work: after an interpolating front-end resampler
        for (auto &s : stage)
            if (!s.p)
                s.alloc(cap);
        if (!ready.p)
            ready.alloc(f->frames_out.n);
        stop = false;
        worker = std::thread([this] { run_worker(); });
        pipelined = true;
    }
    void shutdown_worker()
    {
        if (!worker.joinable())
            return;
        {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return !busy; });
            stop = true;
        }
        cv.notify_all();
        worker.join();
    }
    ~Chain()
    {
        shutdown_worker();
        if (d) {
            DeviceGuard g(d->cfg.device);
            for (cudaEvent_t e : {e0, e1, span0, span1})
                if (e)
                    cudaEventDestroy(e);
        }
        delete d;
        delete f;
    }
};
} // namespace b200
using namespace b200;

struct b200_chain
{
    Chain c;
};

static void chain_push(Chain &c, const void *iq, long n, bool on_device)
{
    B200_REQUIRE(n <= c.d->max_batch, B200_ESTATE, "batch of %ld samples exceeds max_batch %ld", n, c.d->max_batch);
    DeviceGuard g(c.d->cfg.device);
    B200_CUDA(cudaEventRecord(c.e0, c.d->stream));
    // upper bound of the soft bytes this batch can produce
    const double omin = c.d->sps * (1.0 - c.d->cfg.clock_omega_limit) - 0.01;
    const double front = c.d->resamp ? (double)n * c.d->rs_I / c.d->rs_D + 64 : (double)n; // samples after the front-end resampler
    const long bound = (long)(front / omin + 64) * c.d->bps;
    if (c.pipelined) {
        B200_REQUIRE((size_t)bound <= c.stage[c.cur].n, B200_ESTATE, "internal: soft staging buffer too small");
        const long syms = on_device ? c.d->process(iq, n, c.stage[c.cur].p) : c.d->push_host(iq, n, c.stage[c.cur].p);
        std::unique_lock<std::mutex> lk(c.mu);
        c.wait_idle_locked(lk); // the decoder is at most one batch behind
        c.job_bytes = syms * c.d->bps;
        c.job_buf = c.cur;
        c.job_reset = c.reset_pending;
        c.reset_pending = false;
        c.cur ^= 1;
        c.busy = true;
        lk.unlock();
        c.cv.notify_all();
        return;
    }
    B200_REQUIRE(bound <= c.f->append_room(), B200_ESTATE, "decoder soft FIFO too small for this batch (max_soft)");
    long syms;
    if (on_device)
        syms = c.d->process(iq, n, c.f->append_ptr());
    else
        syms = c.d->push_host(iq, n, c.f->append_ptr());
    // the decoder works on its own stream: order it after the demodulator (process() returns synchronised)
    c.f->commit(syms * c.d->bps);
    c.f->process();
    B200_CUDA(cudaEventRecord(c.e1, c.f->stream));
    B200_CUDA(cudaEventSynchronize(c.e1));
    cudaEventElapsedTime(&c.t_total, c.e0, c.e1);
}

// frames of completed batches, oldest first; never waits for the batch in flight. What does not fit into `cap` stays for the next pull.
static long chain_pull(Chain &c, uint8_t *out, long cap)
{
    DeviceGuard g(c.d->cfg.device);
    std::unique_lock<std::mutex> lk(c.mu);
    long nb = 0;
    if (c.ready_frames > 0) {
        nb = c.ready_frames * c.f->cadu_bytes;
        B200_REQUIRE(nb <= cap, B200_ESTATE, "output buffer too small: need %ld bytes", nb);
        B200_CUDA(cudaMemcpyAsync(out, c.ready.p, nb, cudaMemcpyDeviceToHost, c.d->stream));
        B200_CUDA(cudaStreamSynchronize(c.d->stream));
        c.ready_frames = 0;
    }
    // decoder idle: whatever it still holds (synchronous mode, or frames finished while `ready` was occupied)
    if (!c.busy && c.f->out_frames > 0 && (nb == 0 || c.f->out_frames * c.f->cadu_bytes <= cap - nb))
        nb += c.f->pull(out + nb, cap - nb);
    return nb;
}

extern "C" {
b200_chain *b200_chain_create(const b200_demod_cfg *dcfg, const b200_fec_cfg *fcfg)
{
    b200_chain *h = nullptr;
    guarded([&] {
        B200_REQUIRE(dcfg && fcfg, B200_EINVAL, "cfg is NULL");
        B200_REQUIRE(dcfg->device == fcfg->device, B200_EINVAL, "demodulator and decoder of a chain must share a device");
        h = new b200_chain();
        try {
            h->c.d = new Demod(*dcfg);
            // the decoder's soft FIFO must take the soft bytes of a whole demodulated batch whatever the caller guessed: at the
            // lowest samples-per-symbol the clock recovery may settle at (and after an interpolating front-end resampler) that is
            // max_work / omin symbols (e.g. 1.25 soft bytes per sample for QPSK at 1.6 samples per symbol)
            b200_fec_cfg fc = *fcfg;
            const double omin = h->c.d->sps * (1.0 - dcfg->clock_omega_limit) - 0.01;
            const long need = (long)(h->c.d->max_work / omin + 1024) * h->c.d->bps + (1 << 16);
            if (fc.max_soft < need)
                fc.max_soft = need;
            h->c.f = new Fec(fc);
            DeviceGuard g(dcfg->device);
            B200_CUDA(cudaEventCreate(&h->c.e0));
            B200_CUDA(cudaEventCreate(&h->c.e1));
            B200_CUDA(cudaEventCreate(&h->c.span0));
            B200_CUDA(cudaEventCreate(&h->c.span1));
        } catch (...) {
            delete h;
            h = nullptr;
            throw;
        }
    });
    return h;
}
void b200_chain_destroy(b200_chain *h) { delete h; }
int b200_chain_push_iq(b200_chain *h, const void *host_iq, long n)
{
    return guarded([&] {
        B200_REQUIRE(h && host_iq, B200_EINVAL, "NULL argument");
        chain_push(h->c, host_iq, n, false);
    });
}
int b200_chain_push_iq_device(b200_chain *h, const void *dev_iq, long n)
{
    return guarded([&] {
        B200_REQUIRE(h && dev_iq, B200_EINVAL, "NULL argument");
        chain_push(h->c, dev_iq, n, true);
    });
}
int b200_chain_pull_frames(b200_chain *h, uint8_t *out, long cap, long *nbytes)
{
    return guarded([&] {
        B200_REQUIRE(h && out && nbytes, B200_EINVAL, "NULL argument");
        *nbytes = chain_pull(h->c, out, cap);
    });
}
int b200_chain_frames_device(b200_chain *h, const uint8_t **dev_ptr, long *nbytes)
{
    return guarded([&] {
        B200_REQUIRE(h && dev_ptr && nbytes, B200_EINVAL, "NULL argument");
        h->c.sync();
        B200_REQUIRE(h->c.ready_frames == 0, B200_ESTATE, "pipelined chain: pull the pending frames with b200_chain_pull_frames first");
        *dev_ptr = h->c.f->frames_out.p;
        *nbytes = h->c.f->out_frames * h->c.f->cadu_bytes;
        h->c.f->out_frames = 0;
    });
}
int b200_chain_prefetch_iq(b200_chain *h, const void *host_iq, long n)
{
    return guarded([&] {
        B200_REQUIRE(h && host_iq, B200_EINVAL, "NULL argument");
        h->c.d->prefetch_host(host_iq, n);
    });
}
int b200_chain_reset(b200_chain *h)
{
    return guarded([&] {
        B200_REQUIRE(h, B200_EINVAL, "NULL argument");
        if (h->c.pipelined) {
            // the demodulator is idle between pushes; the decoder may still be working on the old stream's last batch: it
            // forgets the stream when the new stream's first batch reaches it. Frames already decoded stay pullable.
            h->c.d->reset();
            std::unique_lock<std::mutex> lk(h->c.mu);
            h->c.reset_pending = true;
            return;
        }
        h->c.d->reset();
        h->c.f->reset();
    });
}
int b200_chain_get_stats(b200_chain *h, b200_demod_stats *ds, b200_fec_stats *fs)
{
    return guarded([&] {
        B200_REQUIRE(h, B200_EINVAL, "NULL argument");
        h->c.sync();
        if (ds)
            h->c.d->stats(ds);
        if (fs)
            h->c.f->stats(fs);
    });
}
int b200_chain_last_timing(b200_chain *h, float *ms, int n)
{
    return guarded([&] {
        B200_REQUIRE(h && ms && n >= 9, B200_EINVAL, "need room for 9 floats");
        Chain &c = h->c;
        c.sync();
        ms[1] = c.d->t_agcfir;
        ms[2] = c.d->t_costas;
        ms[3] = c.d->t_mm;
        ms[4] = c.f->t_vit;
        ms[5] = c.f->t_frames;
        ms[0] = ms[1] + ms[2] + ms[3] + ms[4] + ms[5];
        ms[6] = c.f->t_vit_main;               // k_vit_acs3 alone (sum over its launches in the last push)
        ms[7] = (float)c.f->last_main_chunks;  // chunks those launches decoded
        ms[8] = c.t_total;                     // CUDA-event time from the start of the push (before any H2D) to the last kernel
    });
}
int b200_chain_set_pipelined(b200_chain *h, int on)
{
    return guarded([&] {
        B200_REQUIRE(h, B200_EINVAL, "NULL argument");
        h->c.sync();
        h->c.set_pipelined(on != 0);
    });
}
int b200_chain_sync(b200_chain *h)
{
    return guarded([&] {
        B200_REQUIRE(h, B200_EINVAL, "NULL argument");
        h->c.sync();
    });
}
int b200_chain_span_begin(b200_chain *h)
{
    return guarded([&] {
        B200_REQUIRE(h, B200_EINVAL, "NULL argument");
        Chain &c = h->c;
        c.sync();
        DeviceGuard g(c.d->cfg.device);
        B200_CUDA(cudaStreamSynchronize(c.f->stream));
        B200_CUDA(cudaStreamSynchronize(c.d->stream));
        B200_CUDA(cudaEventRecord(c.span0, c.d->stream));
    });
}
int b200_chain_span_end(b200_chain *h, float *ms)
{
    return guarded([&] {
        B200_REQUIRE(h && ms, B200_EINVAL, "NULL argument");
        Chain &c = h->c;
        c.sync();
        DeviceGuard g(c.d->cfg.device);
        B200_CUDA(cudaStreamSynchronize(c.d->stream));
        B200_CUDA(cudaEventRecord(c.span1, c.f->stream)); // the decoder's stream finishes last
        B200_CUDA(cudaEventSynchronize(c.span1));
        B200_CUDA(cudaEventElapsedTime(ms, c.span0, c.span1));
    });
}
}
