// Host-side plumbing shared by the C-ABI translation units (error text, CUDA checks, device buffers).
#pragma once
#include "../../include/b200dsp.h"
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>

namespace b200
{
void set_error(const char *fmt, ...);

struct ApiError : std::runtime_error
{
    int code;
    ApiError(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

#define B200_CUDA(expr)                                                                                                   \
    do {                                                                                                                  \
        cudaError_t e__ = (expr);                                                                                         \
        if (e__ != cudaSuccess) {                                                                                         \
            char b__[512];                                                                                                \
            snprintf(b__, sizeof(b__), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__);      \
            throw b200::ApiError(B200_ECUDA, b__);                                                                        \
        }                                                                                                                 \
    } while (0)

#define B200_REQUIRE(cond, code, ...)                                                                                     \
    do {                                                                                                                  \
        if (!(cond)) {                                                                                                    \
            char b__[512];                                                                                                \
            snprintf(b__, sizeof(b__), __VA_ARGS__);                                                                      \
            throw b200::ApiError(code, b__);                                                                              \
        }                                                                                                                 \
    } while (0)

template <typename T> struct DevBuf
{
    T *p = nullptr;
    size_t n = 0;
    void alloc(size_t count)
    {
        free();
        if (count == 0)
            count = 1;
        cudaError_t e = cudaMalloc((void **)&p, count * sizeof(T));
        if (e != cudaSuccess) {
            p = nullptr;
            char b[256];
            snprintf(b, sizeof(b), "cudaMalloc of %zu bytes failed: %s", count * sizeof(T), cudaGetErrorString(e));
            throw ApiError(B200_ENOMEM, b);
        }
        n = count;
    }
    void zero(cudaStream_t s) { B200_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), s)); }
    void free()
    {
        if (p)
            cudaFree(p);
        p = nullptr;
        n = 0;
    }
    ~DevBuf() { free(); }
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
};

// DevBuf's counterpart in pinned host memory (the mirrors the device results are copied back into)
template <typename T> struct PinnedBuf
{
    T *p = nullptr;
    size_t n = 0;
    void alloc(size_t count)
    {
        free();
        B200_CUDA(cudaMallocHost((void **)&p, count * sizeof(T)));
        n = count;
    }
    void free()
    {
        if (p)
            cudaFreeHost(p);
        p = nullptr;
        n = 0;
    }
    ~PinnedBuf() { free(); }
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf &) = delete;
    PinnedBuf &operator=(const PinnedBuf &) = delete;
};

// N CUDA events, created by create() and destroyed with the holder
template <int N> struct Events
{
    cudaEvent_t e[N]{};
    void create()
    {
        for (auto &x : e)
            B200_CUDA(cudaEventCreate(&x));
    }
    cudaEvent_t operator[](int i) const { return e[i]; }
    ~Events()
    {
        for (auto &x : e)
            if (x)
                cudaEventDestroy(x);
    }
    Events() = default;
    Events(const Events &) = delete;
    Events &operator=(const Events &) = delete;
};

// selects the device for the calling thread for the lifetime of the guard
struct DeviceGuard
{
    int prev = -1;
    explicit DeviceGuard(int dev)
    {
        cudaGetDevice(&prev);
        if (prev != dev)
            cudaSetDevice(dev);
        else
            prev = -1;
    }
    ~DeviceGuard()
    {
        if (prev >= 0)
            cudaSetDevice(prev);
    }
};

void check_device(int device); // throws B200_ENODEV unless `device` exists and is sm_90

// translate exceptions at the C boundary
template <typename F> int guarded(F &&f)
{
    try {
        f();
        return B200_OK;
    } catch (const ApiError &e) {
        set_error("%s", e.what());
        return e.code;
    } catch (const std::exception &e) {
        set_error("%s", e.what());
        return B200_ECUDA;
    }
}
} // namespace b200
