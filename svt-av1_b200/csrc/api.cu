// api.cu — library management entry points of include/svt_av1_b200.h.
#include <cstdarg>

#include "common.cuh"

namespace svtb200 {
std::atomic<uint64_t> g_launches{0};
static thread_local char t_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_err, sizeof(t_err), fmt, ap);
    va_end(ap);
}
[[noreturn]] void fatal(const char *what, cudaError_t e) {
    fprintf(stderr, "libsvtav1_b200: fatal CUDA error in %s: %s (no CPU fallback)\n", what, cudaGetErrorString(e));
    abort();
}
namespace {
// per-calling-thread stream + growable pinned/device buffers; only Staging reaches them
struct ThreadCtx {
    cudaStream_t stream = nullptr;
    uint8_t *h = nullptr; // pinned
    uint8_t *d = nullptr; // device
    size_t cap = 0;
    int device = -1; // the device stream / d belong to: rebuilt when the calling thread's current device changes
    void free_buffers() {
        if (h) cudaFreeHost(h);
        if (d) cudaFree(d);
        h = d = nullptr;
        cap = 0;
    }
    void drop() {
        free_buffers();
        if (stream) cudaStreamDestroy(stream);
        stream = nullptr;
    }
    // on failure the buffers stay freed (cap 0), so the next call allocates again
    cudaError_t reserve(size_t bytes) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        if (dev != device) { // this thread now serves another GPU: its stream and staging belong to the old one
            if (device >= 0) {
                cudaSetDevice(device);
                drop();
                cudaSetDevice(dev);
            }
            device = dev;
        }
        if (!stream && (e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)) != cudaSuccess) return e;
        if (bytes <= cap) return cudaSuccess;
        size_t ncap = cap ? cap : (1u << 20);
        while (ncap < bytes) ncap *= 2;
        free_buffers();
        void *nh = nullptr, *nd = nullptr;
        if ((e = cudaMallocHost(&nh, ncap)) != cudaSuccess) return e;
        if ((e = cudaMalloc(&nd, ncap)) != cudaSuccess) {
            cudaFreeHost(nh);
            return e;
        }
        h = (uint8_t *)nh, d = (uint8_t *)nd, cap = ncap;
        return cudaSuccess;
    }
    ~ThreadCtx() {
        // the CUDA context may already be gone at thread/process exit; ignore errors
        drop();
    }
};
thread_local ThreadCtx t_ctx;
} // namespace

Staging::Staging(std::initializer_list<size_t> region_bytes) {
    if (region_bytes.size() > kMaxRegions) fatal("Staging: too many regions", cudaErrorInvalidValue);
    size_t o = 0;
    int n = 0;
    for (size_t b : region_bytes) {
        off_[n] = o;
        bytes_[n++] = b;
        o += (b + 255) & ~(size_t)255;
    }
    err_ = t_ctx.reserve(o);
    if (err_ == cudaSuccess) h_ = t_ctx.h, d_ = t_ctx.d, st_ = t_ctx.stream;
}
void Staging::put_rows(int r, const void *src, ptrdiff_t stride, size_t es, size_t width, size_t rows) {
    for (size_t y = 0; y < rows; y++) memcpy(h(r) + y * width * es, (const uint8_t *)src + (ptrdiff_t)y * stride * (ptrdiff_t)es, width * es);
}
void Staging::get_rows(int r, void *dst, ptrdiff_t stride, size_t es, size_t width, size_t rows) const {
    for (size_t y = 0; y < rows; y++) memcpy((uint8_t *)dst + (ptrdiff_t)y * stride * (ptrdiff_t)es, h(r) + y * width * es, width * es);
}
cudaError_t Staging::upload(int first, int last, size_t last_bytes) {
    const size_t n = last_bytes < bytes_[last] ? span(first, last) - bytes_[last] + last_bytes : span(first, last);
    return cudaMemcpyAsync(d(first), h(first), n, cudaMemcpyHostToDevice, st_);
}
cudaError_t Staging::download(int first, int last) {
    const cudaError_t e = cudaMemcpyAsync(h(first), d(first), span(first, last), cudaMemcpyDeviceToHost, st_);
    return e != cudaSuccess ? e : cudaStreamSynchronize(st_);
}
} // namespace svtb200

using namespace svtb200;

extern "C" {
int svt_b200_version(void) { return 100; }
int svt_b200_device_count(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        set_error("cudaGetDeviceCount: %s", cudaGetErrorString(e));
        return e == cudaErrorNoDevice ? 0 : SVT_B200_ERR_CUDA;
    }
    return n;
}
int svt_b200_set_device(int device) {
    SVTB_CUDA_TRY(cudaSetDevice(device));
    return SVT_B200_OK;
}
const char *svt_b200_last_error(void) { return t_err; }
uint64_t svt_b200_launch_count(void) { return g_launches.load(); }
void *svt_b200_malloc(size_t bytes) {
    void *p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) {
        set_error("cudaMalloc(%zu) failed", bytes);
        return nullptr;
    }
    return p;
}
void svt_b200_free(void *p) { cudaFree(p); }
void *svt_b200_malloc_host(size_t bytes) {
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) {
        set_error("cudaMallocHost(%zu) failed", bytes);
        return nullptr;
    }
    return p;
}
void svt_b200_free_host(void *p) { cudaFreeHost(p); }
int svt_b200_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream) {
    SVTB_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return SVT_B200_OK;
}
int svt_b200_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream) {
    SVTB_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    return SVT_B200_OK;
}
int svt_b200_stream_sync(void *stream) {
    SVTB_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
    return SVT_B200_OK;
}
}
