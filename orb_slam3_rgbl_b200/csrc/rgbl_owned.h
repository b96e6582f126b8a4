// Owning handles of the context's CUDA resources (rgbl_ctx.h): device and pinned arrays, streams, events, one graph exec.
// Move-only; each destructor is the one place its resource is released.  The handles convert to the raw pointer / handle
// implicitly, so launches, copies and `buf + offset` arithmetic take them as they took raw pointers.
#ifndef RGBL_OWNED_H
#define RGBL_OWNED_H

#include <cstddef>
#include <utility>

namespace rgbl {

template <class T, bool kPinned>
class OwnedArray {
public:
    OwnedArray() = default;
    OwnedArray(OwnedArray&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    OwnedArray& operator=(OwnedArray&& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
    ~OwnedArray() { reset(); }
    operator T*() const { return p_; }
    T* get() const { return p_; }
    size_t size() const { return n_; }      // elements

    void reset() {
        if (p_) { if constexpr (kPinned) cudaFreeHost(p_); else cudaFree(p_); }
        p_ = nullptr; n_ = 0;
    }
    // exactly n elements, the old array (if any) freed first; on failure the array is empty
    cudaError_t alloc(size_t n) {
        reset();
        cudaError_t e;
        if constexpr (kPinned) e = cudaMallocHost(&p_, n * sizeof(T)); else e = cudaMalloc(&p_, n * sizeof(T));
        if (e != cudaSuccess) { p_ = nullptr; cudaGetLastError(); return e; }
        n_ = n;
        return cudaSuccess;
    }
    // The one reallocation path: at least `need` elements.  A reallocation (contents are not kept) bumps `generation`
    // (Ctx::scratch_generation) and allocates n elements, or need + need / 4 + 64 when n is 0.
    bool grow(size_t need, unsigned long long& generation, size_t n = 0) {
        if (need <= n_) return true;
        ++generation;
        return alloc(n >= need ? n : need + need / 4 + 64) == cudaSuccess;
    }

private:
    T* p_ = nullptr;
    size_t n_ = 0;
};
template <class T> using DeviceArray = OwnedArray<T, false>;
template <class T> using PinnedArray = OwnedArray<T, true>;

// a stream, event or graph exec, released by `Destroy`
template <class H, cudaError_t (*Destroy)(H)>
class OwnedHandle {
public:
    OwnedHandle() = default;
    OwnedHandle(OwnedHandle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    OwnedHandle& operator=(OwnedHandle&& o) noexcept { std::swap(h_, o.h_); return *this; }
    ~OwnedHandle() { reset(); }
    operator H() const { return h_; }
    H get() const { return h_; }
    void reset() { if (h_) Destroy(h_); h_ = nullptr; }

protected:
    // runs a create call that writes the new handle through its argument; on failure the handle stays empty
    template <class F> cudaError_t make(F&& create) {
        reset();
        const cudaError_t e = create(&h_);
        if (e != cudaSuccess) { h_ = nullptr; cudaGetLastError(); }
        return e;
    }

private:
    H h_ = nullptr;
};

struct Stream : OwnedHandle<cudaStream_t, cudaStreamDestroy> {      // non-blocking; priority 0 is the default priority
    cudaError_t create(int priority = 0) { return make([&](cudaStream_t* s) { return cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, priority); }); }
};
struct Event : OwnedHandle<cudaEvent_t, cudaEventDestroy> {
    cudaError_t create(unsigned flags = 0) { return make([&](cudaEvent_t* e) { return cudaEventCreateWithFlags(e, flags); }); }
};
struct GraphExec : OwnedHandle<cudaGraphExec_t, cudaGraphExecDestroy> {
    cudaError_t instantiate(cudaGraph_t graph) { return make([&](cudaGraphExec_t* e) { return cudaGraphInstantiate(e, graph, 0); }); }
};

}  // namespace rgbl
#endif
