// The host frame of a one-shot entry point: the device check, a stream, and the device memory the call allocates.
#pragma once
#include <cuda_runtime.h>

#include "problem_impl.h"

namespace mb200 {

// false + set_error() when no device is usable: the library has no CPU fallback
inline bool have_device()
{
    if(mrcal_b200_device_count() > 0) return true;
    set_error("no usable CUDA device: libmrcal_b200 has no CPU fallback");
    return false;
}

// Every copy and launch of the call goes to `stream`. The destructor drains the stream before it frees the memory, so
// a call that returns early never frees memory under its running kernels or copies
struct DeviceCall
{
    cudaStream_t stream = nullptr;

    DeviceCall() = default;
    DeviceCall(const DeviceCall&) = delete;
    DeviceCall& operator=(const DeviceCall&) = delete;
    ~DeviceCall()
    {
        if(started) cudaStreamSynchronize(stream);
        mem.release();
        if(own) cudaStreamDestroy(stream);
    }

    // the device check, then a non-blocking stream of the call's own
    bool start()
    {
        if(!have_device()) return false;
        MB200_CUDA_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        own = started = true;
        return true;
    }
    // the device check, then the caller's stream: synchronized before the memory is freed, never destroyed
    bool start(cudaStream_t caller)
    {
        if(!have_device()) return false;
        stream = caller;
        started = true;
        return true;
    }

    template <typename T> bool alloc(T** d, size_t n) { return mem.alloc(d, n); }

    // n elements from the host
    template <typename T> bool upload(T** d, const T* h, size_t n)
    {
        if(!mem.alloc(d, n)) return false;
        if(n) MB200_CUDA_CHECK(cudaMemcpyAsync(*d, h, n * sizeof(T), cudaMemcpyHostToDevice, stream));
        return true;
    }
    // rows of w elements, h_pitch bytes apart on the host, packed on the device
    template <typename T> bool upload(T** d, const void* h, size_t h_pitch, size_t w, size_t rows)
    {
        if(!mem.alloc(d, w * rows)) return false;
        if(w && rows)
            MB200_CUDA_CHECK(cudaMemcpy2DAsync(*d, w * sizeof(T), h, h_pitch, w * sizeof(T), rows, cudaMemcpyHostToDevice,
                                               stream));
        return true;
    }
    template <typename T> bool download(T* h, const T* d, size_t n)
    {
        if(n) MB200_CUDA_CHECK(cudaMemcpyAsync(h, d, n * sizeof(T), cudaMemcpyDeviceToHost, stream));
        return true;
    }
    // packed rows of w elements on the device, h_pitch bytes apart on the host
    template <typename T> bool download(void* h, size_t h_pitch, const T* d, size_t w, size_t rows)
    {
        if(w && rows)
            MB200_CUDA_CHECK(cudaMemcpy2DAsync(h, h_pitch, d, w * sizeof(T), w * sizeof(T), rows, cudaMemcpyDeviceToHost,
                                               stream));
        return true;
    }
    // waits for the call's work; false + set_error() if any of it failed
    bool finish()
    {
        MB200_CUDA_CHECK(cudaStreamSynchronize(stream));
        return true;
    }

private:
    DeviceArena mem;
    bool own = false, started = false;
};

}  // namespace mb200
