// Device scratch of the library's synchronous entry points (matching, verification, pose, retrieval, tracks,
// triangulation, bundle adjustment, global poses): one stream-ordered allocation per call from the library's own memory
// pool, laid out in aligned regions, with the host-initialised regions sent in one copy and the allocation freed on every
// exit of the call.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
#include <vector>

namespace psb {

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline unsigned blocks_for(long long n, long long per) { return (unsigned)((n + per - 1) / per); }

// the library's own memory pool of the current device: a pool gives freed memory back to the OS at the next
// synchronisation unless told to keep it, and mapping the workspace again on every call costs more than the matching
// itself (the application's default pool is left alone)
cudaMemPool_t workspace_pool(const char** err);
// Copies device bytes to the host on `st` and waits for the stream
bool read_back(void* dst, const void* src, size_t bytes, cudaStream_t st);

// One call's scratch on stream `st`.  Regions are laid out first (take, put), then allocated at once (alloc); a region's
// offset is its address relative to the allocation (at).  Host bytes given to put or stage are sent by the next upload
// (alloc does one) as a single copy from the first staged byte to the last, with zeros between, through a page-locked
// staging buffer.  The destructor is the only free.
class Workspace {
public:
    // alloc_error, upload_error: what alloc reports when the pool allocation or the upload fails
    Workspace(cudaStream_t st, const char* alloc_error, const char* upload_error)
        : st_(st), alloc_error_(alloc_error), upload_error_(upload_error) {}
    ~Workspace() { if (base_) cudaFreeAsync(base_, st_); }
    Workspace(const Workspace&) = delete;
    Workspace& operator=(const Workspace&) = delete;

    // an uninitialised region of `bytes`, its offset a multiple of `align`
    size_t take(size_t bytes, size_t align = 256);
    // a region holding `bytes` from `src` (nullptr: zeros)
    size_t put(const void* src, size_t bytes, size_t align = 256)
    {
        const size_t off = take(bytes, align);
        stage(off, src, bytes);
        return off;
    }
    // `bytes` from `src` (nullptr: zeros) for the bytes at `off`, sent by the next upload (from the first region staged
    // since the last upload: regions are staged in ascending order)
    void stage(size_t off, const void* src, size_t bytes);
    // the next region is laid out from `off` (regions reused in turn); the allocation covers everything laid out
    void rewind(size_t off) { end_ = off; }
    // the extent of everything laid out so far
    size_t size() const { return size_; }

    // the pool allocation and the upload of the staged bytes; false with *err set on failure
    bool alloc(const char** err);
    // the staged bytes in one copy (none staged: no copy)
    bool upload();
    template <class T>
    T* at(size_t off) const { return reinterpret_cast<T*>(base_ + off); }
    // *err = msg after clearing the last CUDA error; returns -1
    int fail(const char* msg, const char** err) const
    {
        cudaGetLastError();
        *err = msg;
        return -1;
    }

private:
    cudaStream_t st_;
    const char* alloc_error_;
    const char* upload_error_;
    uint8_t* base_ = nullptr;
    size_t end_ = 0, size_ = 0;
    struct Piece { size_t off; std::vector<uint8_t> bytes; };
    bool staged_ = false;
    size_t lo_ = 0, hi_ = 0;        // the span the next upload sends
    std::vector<Piece> pieces_;     // its host bytes, in ascending order
};

} // namespace psb
