// The host rules both translation units of the library share: one error message per thread for b200mvs_last_error and
// b200mvs_depthmap_last_error, one way to fail and to check a CUDA call, the check every *_device entry point makes of
// the caller's buffers (include/b200mvs.h), the wait on the caller's stream, and the camera calibration of a view.
#pragma once
#include "../../include/b200mvs.h"

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>

namespace b200mvs_host {

// The message of the calling thread's last failing call.  Inline, so that both .cu files share the one instance.
inline thread_local std::string last_error;

// Sets the message and returns `code`.  The message is formatted before it is assigned, so `fmt` may read last_error.
inline int fail(int code, const char* fmt, ...)
{
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    last_error = buf;
    return code;
}

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
    return b200mvs_host::fail(B200MVS_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

// Empty when `p` is device or managed memory on `device` and aligned to `align` bytes; else what is wrong with it, to
// follow the buffer's name in an error message.
inline std::string device_buffer_problem(const void* p, int device, size_t align)
{
    cudaPointerAttributes a;
    const cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        cudaGetLastError();                                     // not sticky: keep it from the next call's error check
        return std::string("is not a CUDA pointer (") + cudaGetErrorString(e) + ")";
    }
    if (a.type == cudaMemoryTypeUnregistered) return "is pageable host memory, not device memory";
    if (a.type == cudaMemoryTypeHost) return "is pinned host memory, not device memory";
    if (a.device != device) return "is memory of device " + std::to_string(a.device) + ", not of device " + std::to_string(device);
    if (reinterpret_cast<uintptr_t>(p) % align) return "is not " + std::to_string(align) + "-byte aligned";
    return std::string();
}

// A caller's buffer of a *_device entry point: device (or managed) memory on `device`, aligned to `align` bytes.  0, or
// B200MVS_ERR_INVALID_ARG with a message naming the entry point `fn` and the buffer `what`.
inline int check_device_buffer(const char* fn, const std::string& what, const void* p, int device, size_t align)
{
    const std::string why = device_buffer_problem(p, device, align);
    return why.empty() ? 0 : fail(B200MVS_ERR_INVALID_ARG, "%s: %s %s", fn, what.c_str(), why.c_str());
}

// The work a *_device entry point enqueues on `ours` runs after what the caller enqueued on `caller_stream` (NULL: the
// legacy default stream) before the call; `ev` marks that point.
inline int wait_for_stream(cudaEvent_t ev, void* caller_stream, cudaStream_t ours)
{
    CK(cudaEventRecord(ev, static_cast<cudaStream_t>(caller_stream)));
    CK(cudaStreamWaitEvent(ours, ev, 0));
    return 0;
}

// CameraInfo::fill_calibration / fill_inverse_calibration (camera.cc:125-144,180-200) for an image of width x height
// pixels, in the reference build's arithmetic.  K or Ki may be NULL.
inline void fill_calibration(float flen, float paspect, float ppx, float ppy, float width, float height, float* K, float* Ki)
{
    const float dim_aspect = width / height;
    const float image_aspect = dim_aspect * paspect;
    float ax, ay;
    if (image_aspect < 1.0f) { ax = flen * height / paspect; ay = flen * height; }
    else                     { ax = flen * width;            ay = flen * width * paspect; }
    if (K) {
        K[0] = ax;  K[1] = 0.f; K[2] = width * ppx;
        K[3] = 0.f; K[4] = ay;  K[5] = height * ppy;
        K[6] = 0.f; K[7] = 0.f; K[8] = 1.f;
    }
    if (Ki) {
        Ki[0] = 1.0f / ax; Ki[1] = 0.f;       Ki[2] = -width * ppx / ax;
        Ki[3] = 0.f;       Ki[4] = 1.0f / ay; Ki[5] = -height * ppy / ay;
        Ki[6] = 0.f;       Ki[7] = 0.f;       Ki[8] = 1.f;
    }
}

} // namespace b200mvs_host
