// codec_host.h — host code shared by the codec libraries (libj2pentropy.so, libj2ppng.so,
// libj2pjpegenc.so): J2P_HD, the error buffer, CUDA error checks, the device checks and the encode
// call of the two encoders.  Everything here has internal linkage, so each library keeps its own
// error buffer behind its own j2p_*_last_error and exports nothing new.
#ifndef J2P_CODEC_HOST_H
#define J2P_CODEC_HOST_H

#ifdef __CUDACC__
#define J2P_HD __host__ __device__ __forceinline__
#else
#define J2P_HD static inline
#endif

#include <cuda_runtime.h>

#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <memory>

static thread_local char g_err[256];

static inline int fail(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return -1;
}

#define CK(x)                                                                                   \
    do {                                                                                        \
        const cudaError_t e_ = (x);                                                             \
        if (e_ != cudaSuccess) return fail("%s: %s", #x, cudaGetErrorString(e_));               \
    } while (0)

static inline size_t align16(size_t n) { return (n + 15) & ~(size_t)15; }

static inline int device_of(const void *ptr, const char *what, int *dev) {
    cudaPointerAttributes a;
    const cudaError_t e = cudaPointerGetAttributes(&a, ptr);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail("%s: %s", what, cudaGetErrorString(e));
    }
    if (a.type != cudaMemoryTypeDevice) return fail("%s is not device memory", what);
    *dev = a.device;
    return 0;
}

struct DeviceGuard {
    int prev = -1;
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// *dev: the device of the work area, after checking that it and every image's data are device
// memory on that one device
template <class Image>
static int same_device(const Image *images, unsigned n, const void *work, int *dev) {
    if (device_of(work, "the work area", dev) != 0) return -1;
    for (unsigned i = 0; i < n; i++) {
        char what[48];
        int d = -1;
        snprintf(what, sizeof what, "image %u's data", i);
        if (device_of(images[i].data, what, &d) != 0) return -1;
        if (d != *dev) return fail("image %u is on device %d, the work area on device %d", i, d, *dev);
    }
    return 0;
}

// One device encode call of libj2ppng.so or libj2pjpegenc.so, after the caller's plan L has
// accepted the images: checks the arguments and the devices, fills the first plan_bytes of the work
// area on the host (fill(plan) -> 0 or fail) and uploads them, queues the kernels on the work area's
// device (launch(w, stream, plan, counted) -> 0 or fail, calling counted() after each launch), reads
// back the n + 1 file offsets, waits for the stream and copies the files into dst when it is given.
// stats->launches gets the kernels queued without a launch error.
template <class Image, class Layout, class Stats, class Fill, class Launch>
static int encode_call(const Image *images, unsigned n, const Layout &L, size_t plan_bytes, void *work, size_t work_bytes, void *stream,
                       uint64_t *offsets, void *dst, size_t dst_cap, Stats *stats, Fill fill, Launch launch) {
    if (!work || !offsets) return fail("null argument");
    if (work_bytes < L.total) return fail("work area of %zu bytes is smaller than the plan's %zu", work_bytes, L.total);
    int dev = -1;
    if (same_device(images, n, work, &dev) != 0) return -1;
    DeviceGuard guard;
    CK(cudaGetDevice(&guard.prev));
    CK(cudaSetDevice(dev));
    const cudaStream_t st = (cudaStream_t)stream;
    // freed on return: on the normal path only after the stream synchronise, when the upload has read it
    const std::unique_ptr<uint8_t, decltype(&free)> plan((uint8_t *)malloc(plan_bytes), &free);
    if (!plan) return fail("out of host memory");
    if (fill(plan.get()) != 0) return -1;
    uint8_t *w = (uint8_t *)work;
    const cudaError_t ec = cudaMemcpyAsync(w, plan.get(), plan_bytes, cudaMemcpyHostToDevice, st);
    if (ec != cudaSuccess) return fail("plan upload: %s", cudaGetErrorString(ec));
    unsigned launches = 0;
    auto counted = [&]() { launches += cudaPeekAtLastError() == cudaSuccess; };
    if (launch(w, st, (const uint8_t *)plan.get(), counted) != 0) return -1;
    const cudaError_t el = cudaGetLastError();
    if (el != cudaSuccess) return fail("launch: %s", cudaGetErrorString(el));
    const cudaError_t eo = cudaMemcpyAsync(offsets, w + L.off_offs, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
    const cudaError_t es = eo == cudaSuccess ? cudaStreamSynchronize(st) : eo;
    if (es != cudaSuccess) return fail("encode: %s", cudaGetErrorString(es));
    if (dst) {
        if (dst_cap < offsets[n]) return fail("destination of %zu bytes is smaller than the files (%llu)", dst_cap, (unsigned long long)offsets[n]);
        CK(cudaMemcpyAsync(dst, w + L.off_out, offsets[n], cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    if (stats) stats->launches = launches;
    return 0;
}

#endif  // J2P_CODEC_HOST_H
