// seal_b200/csrc/sb_mem.cuh -- owners of the device memory, page-locked staging, streams and events of a context and its keys.
// Destroying an owner releases what it holds, so the device that holds it must be current then: the destructors of Context and of
// the key handles select it in their bodies, before their members are destroyed.  Kernel-facing structs (PrimeDev, Src, the Op
// functors) keep raw pointers: they are views of memory owned here.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <memory>
#include <stdexcept>
#include <type_traits>
#include <utility>

namespace sb
{
    struct CudaError : std::runtime_error
    {
        using std::runtime_error::runtime_error;
    };
    void cuda_check(cudaError_t e, const char *what);

    // count elements of T in device memory (PINNED: page-locked host memory), move-only.  With wipe set the memory is zeroed
    // before it is freed: secret material never goes back to the allocator in clear (the reference keeps secret keys in
    // clear-on-destruction pools, secretkey.h:51-60).
    template <class T, bool PINNED = false>
    class DevBuf
    {
    public:
        DevBuf() = default;
        explicit DevBuf(size_t count, bool wipe = false) : wipe_(wipe)
        {
            if (!count)
                return;
            void *p = nullptr;
            if constexpr (PINNED)
                cuda_check(cudaHostAlloc(&p, count * sizeof(T), cudaHostAllocDefault), "cudaHostAlloc");
            else
                cuda_check(cudaMalloc(&p, count * sizeof(T)), "cudaMalloc");
            p_ = static_cast<T *>(p), bytes_ = count * sizeof(T);
        }
        DevBuf(DevBuf &&o) noexcept : p_(std::exchange(o.p_, nullptr)), bytes_(std::exchange(o.bytes_, 0)), wipe_(o.wipe_) {}
        DevBuf &operator=(DevBuf &&o) noexcept
        {
            if (this != &o)
            {
                release();
                p_ = std::exchange(o.p_, nullptr), bytes_ = std::exchange(o.bytes_, 0), wipe_ = o.wipe_;
            }
            return *this;
        }
        ~DevBuf() { release(); }

        T *get() const { return p_; }
        size_t bytes() const { return bytes_; }
        explicit operator bool() const { return p_ != nullptr; }

        // the grow-only arenas: room for at least count elements.  Growing first waits for the device, whose work in flight may
        // still use the old memory.  The old memory is released before the new is allocated, unless keep asks for its contents at
        // the front of the new memory.
        void grow(size_t count, bool keep = false)
        {
            if (count * sizeof(T) <= bytes_)
                return;
            cuda_check(cudaDeviceSynchronize(), "sync before arena growth");
            if (!keep)
                release();
            DevBuf grown(count, wipe_);
            if (p_)
                cuda_check(cudaMemcpy(grown.p_, p_, bytes_, cudaMemcpyDefault), "copy before arena growth");
            *this = std::move(grown);
        }

    private:
        void release() noexcept
        {
            if (!p_)
                return;
            if (wipe_)
            {
                cudaMemset(p_, 0, bytes_);
                cudaDeviceSynchronize();
            }
            if constexpr (PINNED)
                cudaFreeHost(p_);
            else
                cudaFree(p_);
            p_ = nullptr, bytes_ = 0;
        }

        T *p_ = nullptr;
        size_t bytes_ = 0;
        bool wipe_ = false;
    };
    using PinnedBuf = DevBuf<unsigned char, true>;

    struct StreamDestroy
    {
        void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
    };
    struct EventDestroy
    {
        void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
    };
    using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDestroy>;
    using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDestroy>;

    inline Stream make_stream()
    {
        cudaStream_t s = nullptr;
        cuda_check(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking), "cudaStreamCreate");
        return Stream(s);
    }
    inline Event make_event()
    {
        cudaEvent_t e = nullptr;
        cuda_check(cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "cudaEventCreate");
        return Event(e);
    }
} // namespace sb
