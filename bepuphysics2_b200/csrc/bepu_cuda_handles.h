// Host-side owners of the CUDA resources the solver context and its drivers hold (bepucuda_api.cu, bepu_coloring.cu, bepu_islands.cu): each frees
// its resource in its destructor, so no resource needs a hand-written release list. Host code only.
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <cstddef>
#include <utility>
#include <vector>

namespace bepucuda {

// Memory that grows on demand (contents are not kept) and is freed with its owner: device memory, or page-locked host memory.
template <bool kPinnedHost> struct GrowBuffer {
    void* ptr = nullptr;
    size_t capacity = 0;
    GrowBuffer() = default;
    GrowBuffer(const GrowBuffer&) = delete;
    GrowBuffer& operator=(const GrowBuffer&) = delete;
    ~GrowBuffer() { release(); }
    cudaError_t reserve(size_t bytes) {
        if (bytes <= capacity) return cudaSuccess;
        release();
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = kPinnedHost ? cudaMallocHost(&ptr, want) : cudaMalloc(&ptr, want);
        if (e == cudaSuccess) capacity = want;
        else ptr = nullptr;
        return e;
    }
    // Device memory only: room for `bytes` with the first `keep` bytes kept (a stream-ordered device copy into a block of at least twice the
    // capacity, so that repeated growth copies each byte a bounded number of times). On failure the buffer is as it was.
    cudaError_t grow(size_t bytes, size_t keep, cudaStream_t s) {
        static_assert(!kPinnedHost, "grow keeps device memory");
        if (bytes <= capacity) return cudaSuccess;
        const size_t want = std::max(bytes, 2 * capacity);
        void* n = nullptr;
        cudaError_t e = cudaMalloc(&n, want);
        if (e == cudaSuccess && keep > 0) e = cudaMemcpyAsync(n, ptr, std::min(keep, capacity), cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) {
            if (n) cudaFree(n);
            return e;
        }
        release();  // cudaFree waits for the copy
        ptr = n;
        capacity = want;
        return cudaSuccess;
    }
    void release() {
        if (ptr) kPinnedHost ? cudaFreeHost(ptr) : cudaFree(ptr);
        ptr = nullptr;
        capacity = 0;
    }
    template <class T> T* as() const { return (T*)ptr; }
};
using DeviceBuffer = GrowBuffer<false>;
using PinnedBuffer = GrowBuffer<true>;

// Bump allocator over chunks that are never reallocated (uploads are enqueued against their addresses).
struct ChunkArena {
    struct Chunk { char* base; size_t size, used; };
    std::vector<Chunk> chunks;
    bool pinned_host = false;
    size_t min_chunk = (size_t)64 << 20;
    ChunkArena() = default;
    ChunkArena(const ChunkArena&) = delete;
    ChunkArena& operator=(const ChunkArena&) = delete;
    ~ChunkArena() {
        for (auto& c : chunks) { if (pinned_host) cudaFreeHost(c.base); else cudaFree(c.base); }
    }
    void reset() { for (auto& c : chunks) c.used = 0; }
    void* alloc(size_t bytes, cudaError_t* err) {
        bytes = (bytes + 255) & ~(size_t)255;
        for (auto& c : chunks)
            if (c.size - c.used >= bytes) {
                void* p = c.base + c.used;
                c.used += bytes;
                return p;
            }
        Chunk c{};
        c.size = std::max(bytes, min_chunk);
        cudaError_t e = pinned_host ? cudaMallocHost((void**)&c.base, c.size) : cudaMalloc((void**)&c.base, c.size);
        if (e != cudaSuccess) { if (err) *err = e; return nullptr; }
        c.used = bytes;
        chunks.push_back(c);
        return chunks.back().base;
    }
};

// One CUDA handle, released by kRelease when its owner is reset or destroyed. Movable, not copyable; reads as the raw handle.
template <class T, cudaError_t (*kRelease)(T)> struct Owned {
    T h_ = nullptr;
    Owned() = default;
    Owned(Owned&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    Owned& operator=(Owned&& o) noexcept { std::swap(h_, o.h_); return *this; }
    ~Owned() { reset(); }
    void reset() { if (h_) kRelease(std::exchange(h_, nullptr)); }
    T* put() { reset(); return &h_; }  // the out-parameter of the call that creates the handle
    operator T() const { return h_; }
};
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Graph = Owned<cudaGraph_t, cudaGraphDestroy>;
using GraphExec = Owned<cudaGraphExec_t, cudaGraphExecDestroy>;
using IpcMapping = Owned<void*, cudaIpcCloseMemHandle>;  // a peer allocation opened by cudaIpcOpenMemHandle
// A CUDA event, created with the flags of the site that uses it.
struct Event : Owned<cudaEvent_t, cudaEventDestroy> {
    cudaError_t create(unsigned flags = cudaEventDefault) { return h_ ? cudaSuccess : cudaEventCreateWithFlags(&h_, flags); }  // no-op once created
};

// Pinned copy of a host buffer that the caller may reuse as soon as the upload is enqueued, and the event after which the copy has read it.
struct StagedUpload {
    PinnedBuffer host;
    Event done;
};

// A stream interval timed by two events: measured once it has been closed, until it is opened again.
struct TimingWindow {
    Event begin, end;
    bool open = false, recorded = false;
    cudaError_t start(cudaStream_t s) { open = true; return cudaEventRecord(begin, s); }
    void start_once(cudaStream_t s) { if (!open) start(s); }  // an upload window spans every upload until the next frame
    cudaError_t stop(cudaStream_t s) { open = false; recorded = true; return cudaEventRecord(end, s); }
    void measure(float* ms) const { if (recorded && !open) cudaEventElapsedTime(ms, begin, end); }
};

}  // namespace bepucuda
