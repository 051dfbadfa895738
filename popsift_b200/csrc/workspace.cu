// Device scratch of the synchronous entry points (workspace.h).
#include "workspace.h"
#include "k_match_plan.h"

#include <algorithm>
#include <cassert>
#include <cstring>
#include <mutex>

namespace psb {

cudaMemPool_t workspace_pool(const char** err)
{
    static std::mutex mu;
    static cudaMemPool_t pools[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { cudaGetLastError(); *err = "cudaGetDevice failed (matcher)"; return nullptr; }
    std::lock_guard<std::mutex> g(mu);
    if (!pools[dev]) {
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.handleTypes = cudaMemHandleTypeNone;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = dev;
        if (cudaMemPoolCreate(&pools[dev], &props) != cudaSuccess) { cudaGetLastError(); pools[dev] = nullptr; *err = "cudaMemPoolCreate failed (matcher)"; return nullptr; }
        unsigned long long keep = kMatchPoolKeep;                              // freed workspace that stays mapped
        cudaMemPoolSetAttribute(pools[dev], cudaMemPoolAttrReleaseThreshold, &keep);
    }
    return pools[dev];
}

namespace {

// Copies `bytes` to `dst` on `st` from a page-locked staging buffer of the current device, which fill(buffer) writes, so
// that the copy is queued without waiting (a pageable source would hold the host until the transfer is done).  The
// buffer is reused by the next call once the event recorded after this copy has completed.
template <class Fill>
bool upload_plan(void* dst, size_t bytes, Fill fill, cudaStream_t st)
{
    struct Stage { uint8_t* buf = nullptr; size_t cap = 0; cudaEvent_t done = nullptr; };
    static std::mutex mu;
    static Stage stages[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { cudaGetLastError(); return false; }
    std::lock_guard<std::mutex> g(mu);
    Stage& s = stages[dev];
    if (!s.done && cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); s.done = nullptr; return false; }
    if (cudaEventSynchronize(s.done) != cudaSuccess) { cudaGetLastError(); return false; }     // the previous copy has left the buffer
    if (s.cap < bytes) {
        if (s.buf) cudaFreeHost(s.buf);
        s.buf = nullptr; s.cap = 0;
        const size_t cap = std::max<size_t>(align_up(bytes, 1 << 16), 1 << 16);
        if (cudaHostAlloc(reinterpret_cast<void**>(&s.buf), cap, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); s.buf = nullptr; return false; }
        s.cap = cap;
    }
    fill(s.buf);
    if (cudaMemcpyAsync(dst, s.buf, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) { cudaGetLastError(); return false; }
    if (cudaEventRecord(s.done, st) != cudaSuccess) { cudaGetLastError(); return false; }
    return true;
}

} // namespace

bool read_back(void* dst, const void* src, size_t bytes, cudaStream_t st)
{
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st) == cudaSuccess && cudaStreamSynchronize(st) == cudaSuccess;
}

size_t Workspace::take(size_t bytes, size_t align)
{
    const size_t off = align_up(end_, align);
    end_ = off + bytes;
    size_ = std::max(size_, end_);
    return off;
}

void Workspace::stage(size_t off, const void* src, size_t bytes)
{
    if (!staged_) {
        staged_ = true;
        lo_ = hi_ = off;
    }
    assert(off >= hi_ || bytes == 0);
    hi_ = std::max(hi_, off + bytes);
    if (src && bytes) pieces_.push_back({off, std::vector<uint8_t>(static_cast<const uint8_t*>(src), static_cast<const uint8_t*>(src) + bytes)});
}

bool Workspace::alloc(const char** err)
{
    cudaMemPool_t pool = workspace_pool(err);
    if (!pool) return false;
    // stream-ordered, so nothing blocks; the allocation ends on a 256-byte boundary
    if (cudaMallocFromPoolAsync(&base_, align_up(size_, 256), pool, st_) != cudaSuccess) {
        base_ = nullptr;
        fail(alloc_error_, err);
        return false;
    }
    if (!upload()) {
        fail(upload_error_, err);
        return false;
    }
    return true;
}

bool Workspace::upload()
{
    if (!staged_) return true;
    // the pieces in ascending order, zeros between them
    const bool ok = upload_plan(base_ + lo_, hi_ - lo_, [this](uint8_t* buf) {
        size_t at = lo_;
        for (const Piece& p : pieces_) {
            std::memset(buf + (at - lo_), 0, p.off - at);
            std::memcpy(buf + (p.off - lo_), p.bytes.data(), p.bytes.size());
            at = p.off + p.bytes.size();
        }
        std::memset(buf + (at - lo_), 0, hi_ - at);
    }, st_);
    staged_ = false;
    pieces_.clear();
    return ok;
}

} // namespace psb
