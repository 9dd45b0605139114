// immesh_b200 -- the one owner of device and pinned host memory in the host code of the handles.  A MemSet holds blocks that
// are all from cudaMalloc (Device) or all from cudaMallocHost (Pinned), knows their byte total and frees every block it still
// holds when it is destroyed.  Each block is one allocation call, with the size the caller asked for: there is no pooling or
// sub-allocation.  Host code only, so that it builds without nvcc.
#pragma once
#include <cuda_runtime_api.h>

#include <algorithm>
#include <cassert>
#include <cstddef>
#include <cstring>
#include <utility>
#include <vector>

namespace immesh {

class MemSet {
  public:
    enum Kind { Device, Pinned };
    MemSet() = default;
    explicit MemSet(Kind kind) : kind_(kind) {}
    MemSet(MemSet&& o) noexcept : kind_(o.kind_), blocks_(std::move(o.blocks_)) { o.blocks_.clear(); }
    MemSet& operator=(MemSet&& o) noexcept {
        if (this != &o) {
            release();
            kind_ = o.kind_;
            blocks_ = std::move(o.blocks_);
            o.blocks_.clear();
        }
        return *this;
    }
    MemSet(const MemSet&) = delete;
    MemSet& operator=(const MemSet&) = delete;
    ~MemSet() { release(); }

    // one block of `count` T, filled with `memset_byte` when it is >= 0.  On failure *p is untouched and the set unchanged.
    template <class T>
    cudaError_t alloc(T** p, size_t count, int memset_byte = -1) {
        const size_t bytes = count * sizeof(T);
        void* q = nullptr;
        cudaError_t e = kind_ == Pinned ? cudaMallocHost(&q, bytes) : cudaMalloc(&q, bytes);
        if (e != cudaSuccess) return e;
        if (memset_byte >= 0) {
            if (kind_ == Pinned) std::memset(q, memset_byte, bytes);
            else if ((e = cudaMemset(q, memset_byte, bytes)) != cudaSuccess) { free_block(q); return e; }
        }
        blocks_.push_back({q, bytes});
        *p = static_cast<T*>(q);
        return cudaSuccess;
    }
    // frees block p of the set (null, or a pointer the set does not hold: nothing)
    void free(const void* p) {
        for (size_t i = 0; p && i < blocks_.size(); ++i) {
            if (blocks_[i].p != p) continue;
            free_block(blocks_[i].p);
            blocks_.erase(blocks_.begin() + i);
            return;
        }
    }
    // every block of `o` joins this set (same kind)
    void take(MemSet&& o) {
        assert(o.kind_ == kind_);
        blocks_.insert(blocks_.end(), o.blocks_.begin(), o.blocks_.end());
        o.blocks_.clear();
    }
    // grow-only scratch of *cap T at *p: when need > *cap, the old block is freed first and max(need, floor) T are allocated.
    // On failure *p is null and *cap 0, so that the next call tries again.
    template <class T>
    cudaError_t regrow(T** p, size_t* cap, size_t need, size_t floor = 0) {
        if (need <= *cap) return cudaSuccess;
        free(*p);
        *p = nullptr;
        *cap = 0;
        const size_t c = std::max(need, floor);
        const cudaError_t e = alloc(p, c);
        if (e == cudaSuccess) *cap = c;
        return e;
    }
    size_t bytes() const {
        size_t s = 0;
        for (const Block& b : blocks_) s += b.bytes;
        return s;
    }

  private:
    struct Block { void* p; size_t bytes; };
    void free_block(void* p) const {
        if (kind_ == Pinned) cudaFreeHost(p);
        else cudaFree(p);
    }
    void release() {
        for (const Block& b : blocks_) free_block(b.p);
        blocks_.clear();
    }
    Kind kind_ = Device;
    std::vector<Block> blocks_;
};

}  // namespace immesh
