// Owners of the host side's CUDA resources (rt_kernels.cu).  The kernels keep taking raw pointers and handles; these types only
// decide when the resources behind them are released.
#pragma once

#include <cuda_runtime.h>

#include <memory>
#include <type_traits>
#include <vector>

// Device (and pinned host) allocations that share one lifetime: all freed by clear() and by the destructor.  A group is built
// in a local and moved into its place once every allocation has succeeded, so a failure leaves the previous state as it was.
class DevAllocs
{
public:
    DevAllocs() = default;
    DevAllocs(DevAllocs&& o) noexcept { blocks_.swap(o.blocks_); }
    DevAllocs& operator=(DevAllocs&& o) noexcept { if (this != &o) { clear(); blocks_.swap(o.blocks_); } return *this; }
    ~DevAllocs() { clear(); }

    // count elements of T, in device memory or (host) pinned host memory; the view, the raw pointer the kernels take, is set
    // only on success
    template <class T> cudaError_t alloc(T*& view, size_t count, bool host = false)
    {
        void* p = nullptr;
        const cudaError_t e = host ? cudaMallocHost(&p, count * sizeof(T)) : cudaMalloc(&p, count * sizeof(T));
        if (e == cudaSuccess) { blocks_.push_back({ p, host }); view = (T*)p; }
        return e;
    }
    // takes over o's allocations (a part of this group that was built on its own)
    void adopt(DevAllocs&& o) { blocks_.insert(blocks_.end(), o.blocks_.begin(), o.blocks_.end()); o.blocks_.clear(); }
    void clear() { for (const Block& b : blocks_) b.host ? cudaFreeHost(b.p) : cudaFree(b.p); blocks_.clear(); }
    bool empty() const { return blocks_.empty(); }

private:
    struct Block { void* p; bool host; };
    std::vector<Block> blocks_;
};

struct CudaDestroy
{
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
    void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
    void operator()(cudaGraph_t g) const { cudaGraphDestroy(g); }
    void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); }
};

// A stream, event or graph that destroys itself.  It converts to the raw handle, so it is passed to the runtime as it is.
template <class H> struct Owned : std::unique_ptr<std::remove_pointer_t<H>, CudaDestroy>
{
    using std::unique_ptr<std::remove_pointer_t<H>, CudaDestroy>::unique_ptr;
    operator H() const { return this->get(); }
};

inline cudaError_t make_stream(Owned<cudaStream_t>& s)
{
    cudaStream_t h = nullptr;
    const cudaError_t e = cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking);
    if (e == cudaSuccess) s.reset(h);
    return e;
}

inline cudaError_t make_event(Owned<cudaEvent_t>& ev, unsigned flags = cudaEventDisableTiming)
{
    cudaEvent_t h = nullptr;
    const cudaError_t e = cudaEventCreateWithFlags(&h, flags);
    if (e == cudaSuccess) ev.reset(h);
    return e;
}

// owns a mapping of another process's buffer (rt_ipc_open)
struct IpcClose { void operator()(void* p) const { cudaIpcCloseMemHandle(p); } };
