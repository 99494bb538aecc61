// The check every *_device entry point makes of the caller's buffers before it runs anything (include/b200mvs.h).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

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
