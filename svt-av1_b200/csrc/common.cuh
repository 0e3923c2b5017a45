// common.cuh — shared infrastructure of libsvtav1_b200.so (sm_90a only).
//  * error capture (thread-local message, negative SvtB200Status codes, no CPU fallback)
//  * launch counter (svt_b200_launch_count)
//  * Staging: the regions of one host-pointer call in the calling thread's stream + growable pinned/device
//    buffers.  The RTCD drop-ins — like the reference's function pointers (SURVEY §8b) — are re-entrant and
//    called concurrently from every pipeline thread with raw host pointers.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>

#include "../../include/svt_av1_b200.h"

namespace svtb200 {

extern std::atomic<uint64_t> g_launches;
void set_error(const char *fmt, ...);

#define SVTB_CUDA_TRY(expr)                                                                   \
    do {                                                                                      \
        cudaError_t e__ = (expr);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            svtb200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return SVT_B200_ERR_CUDA;                                                         \
        }                                                                                     \
    } while (0)

// Launch + count. Use as: SVTB_LAUNCH(kernel, grid, block, smem, stream, args...)
#define SVTB_LAUNCH(kern, grid, block, smem, stream, ...)           \
    do {                                                            \
        kern<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);   \
        svtb200::g_launches.fetch_add(1, std::memory_order_relaxed); \
    } while (0)

// A drop-in has no error return (the reference's kernels return void): a CUDA failure is fatal, exactly
// like EB_ErrorMax through lib_svt_encoder_send_error_exit — log and abort; never fall back to the CPU.
[[noreturn]] void fatal(const char *what, cudaError_t e);
#define SVTB_CUDA_FATAL(expr)                            \
    do {                                                 \
        cudaError_t e__ = (expr);                        \
        if (e__ != cudaSuccess) svtb200::fatal(#expr, e__); \
    } while (0)

// The staging of one host-pointer call (the RTCD drop-ins and the `_host` entries) on the calling thread's stream and
// its pinned + device buffers.  A call names its regions in order with their byte sizes; every region starts on a
// 256-byte boundary, so a kernel that reads a little past the end of its region stays inside the buffers.  The
// constructor reserves the buffers once, before any region is written; a reservation can move them, so nothing the
// call runs while it holds region pointers may construct another Staging on the same thread.
class Staging {
  public:
    Staging(std::initializer_list<size_t> region_bytes);
    // the reservation's error, if any: the thread's buffers are then empty and its next call allocates again
    cudaError_t status() const { return err_; }
    cudaStream_t stream() const { return st_; }
    template <typename T = uint8_t>
    T *h(int r) const { return reinterpret_cast<T *>(h_ + off_[r]); }
    template <typename T = uint8_t>
    T *d(int r) const { return reinterpret_cast<T *>(d_ + off_[r]); }
    size_t off(int r) const { return off_[r]; }
    size_t span(int first, int last) const { return off_[last] + bytes_[last] - off_[first]; }
    // `rows` rows of `width` elements of `es` bytes, `stride` elements apart from `src`, packed into region r
    void put_rows(int r, const void *src, ptrdiff_t stride, size_t es, size_t width, size_t rows);
    // the packed rows of region r out to `dst`, `stride` elements apart
    void get_rows(int r, void *dst, ptrdiff_t stride, size_t es, size_t width, size_t rows) const;
    // one copy of regions first..last to the device; of the last region only its first `last_bytes`
    cudaError_t upload(int first, int last, size_t last_bytes = SIZE_MAX);
    // one copy of regions first..last to the host, then a wait for the stream
    cudaError_t download(int first, int last);

  private:
    static constexpr int kMaxRegions = 16;
    size_t off_[kMaxRegions], bytes_[kMaxRegions];
    uint8_t *h_ = nullptr, *d_ = nullptr;
    cudaStream_t st_ = nullptr;
    cudaError_t err_;
};

// Per-DEVICE one-time set-up (cudaFuncSetAttribute, occupancy queries and table uploads are per device, a process may
// use several - svt_b200_set_device): `fn` runs once for the calling thread's current device, under a lock, and its
// CUDA errors are fatal (no CPU fallback).  Usage: static PerDeviceOnce once; once.run([]{ ... });
struct PerDeviceOnce {
    std::atomic<int> done[64];
    PerDeviceOnce() {
        for (auto &d : done) d.store(0);
    }
    template <typename F>
    void run(F fn) {
        int dev = 0;
        SVTB_CUDA_FATAL(cudaGetDevice(&dev));
        dev &= 63;
        if (done[dev].load(std::memory_order_acquire) == 2) return;
        int expect = 0;
        if (done[dev].compare_exchange_strong(expect, 1)) {
            fn();
            done[dev].store(2, std::memory_order_release);
        } else {
            while (done[dev].load(std::memory_order_acquire) != 2) {
            } // another pipeline thread is setting this device up
        }
    }
};
#define SVTB_ATTR(kernel, bytes) SVTB_CUDA_FATAL(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes))

// ---- device helpers -------------------------------------------------------------------------------
// 4 byte-wise absolute differences accumulated into acc (PTX vabsdiff4 with the .add merge).
__device__ __forceinline__ uint32_t sad4(uint32_t a, uint32_t b, uint32_t acc) {
    uint32_t d;
    asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(acc));
    return d;
}
__device__ __forceinline__ uint64_t warp_min_u64(uint64_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        uint64_t w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w < v ? w : v;
    }
    return v;
}
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

} // namespace svtb200
