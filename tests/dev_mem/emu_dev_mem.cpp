// Host harness of immesh_b200/csrc/dev_mem.hpp: the CUDA allocation calls it makes are defined here, backed by malloc, with
// every live block tracked by kind and a switch that makes the k-th allocation (or a memset) fail.  Each dm_* scenario runs one
// use of MemSet the handles rely on and returns 0, or the line of the first check that failed.
#include <cstdlib>
#include <cstring>
#include <map>
#include <utility>

#include "../../immesh_b200/csrc/dev_mem.hpp"

namespace {
enum Kind { Dev = 0, Host = 1 };
std::map<void*, Kind> g_live;   // block -> how it was allocated
long long g_allocs = 0;         // allocation calls so far
long long g_fail_at = 0;        // the allocation call that fails (1-based; 0: none)
int g_memset_fail = 0;          // cudaMemset fails
int g_misuse = 0;               // frees of an unknown block, or with the other kind's call
long long g_seq = 0, g_last_free_seq = 0, g_last_alloc_seq = 0;   // order of the calls

cudaError_t stub_alloc(void** p, size_t bytes, Kind k) {
    ++g_allocs;
    if (g_fail_at && g_allocs == g_fail_at) return cudaErrorMemoryAllocation;
    void* q = std::malloc(bytes ? bytes : 1);
    g_live[q] = k;
    *p = q;
    g_last_alloc_seq = ++g_seq;
    return cudaSuccess;
}
cudaError_t stub_free(void* p, Kind k) {
    if (!p) return cudaSuccess;
    auto it = g_live.find(p);
    if (it == g_live.end() || it->second != k) { ++g_misuse; return cudaErrorInvalidValue; }
    g_live.erase(it);
    std::free(p);
    g_last_free_seq = ++g_seq;
    return cudaSuccess;
}
long long live(Kind k) {
    long long n = 0;
    for (const auto& b : g_live) n += b.second == k;
    return n;
}
}  // namespace

extern "C" {
cudaError_t cudaMalloc(void** p, size_t bytes) { return stub_alloc(p, bytes, Dev); }
cudaError_t cudaMallocHost(void** p, size_t bytes) { return stub_alloc(p, bytes, Host); }
cudaError_t cudaFree(void* p) { return stub_free(p, Dev); }
cudaError_t cudaFreeHost(void* p) { return stub_free(p, Host); }
cudaError_t cudaMemset(void* p, int value, size_t bytes) {
    if (g_memset_fail) return cudaErrorInvalidValue;
    auto it = g_live.find(p);
    if (it == g_live.end() || it->second != Dev) { ++g_misuse; return cudaErrorInvalidValue; }
    std::memset(p, value, bytes);
    return cudaSuccess;
}

// the harness state: allocation calls, live device / pinned blocks, misuse count
void dm_reset(long long fail_at) {
    g_allocs = 0;
    g_fail_at = fail_at;
    g_memset_fail = 0;
}
long long dm_allocs() { return g_allocs; }
long long dm_live(int pinned) { return live(pinned ? Host : Dev); }
int dm_misuse() { return g_misuse; }

#define CHECK(c) do { if (!(c)) return __LINE__; } while (0)
using immesh::MemSet;

// growth-shaped transaction: the handle's set holds a and b (plus c, which stays); a local set allocates the replacements of a and
// b and a temporary; on success a and b are freed from the handle's set and the local set is taken into it.  The allocation calls
// of the transaction are numbered from 1 (the handle's own blocks are allocated before the failure switch is set).
int dm_transaction(long long fail_at) {
    dm_reset(0);
    {
        MemSet own;
        double* a = nullptr;
        int* b = nullptr;
        char* c = nullptr;
        CHECK(own.alloc(&a, 10) == cudaSuccess && own.alloc(&b, 20) == cudaSuccess && own.alloc(&c, 3) == cudaSuccess);
        CHECK(own.bytes() == 80 + 80 + 3 && live(Dev) == 3);
        dm_reset(fail_at);
        bool ok = false;
        {
            MemSet fresh, tmp;
            double* a2 = a;
            int* b2 = b;
            long long* t = nullptr;
            cudaError_t e;
            if ((e = fresh.alloc(&a2, 40)) == cudaSuccess && (e = fresh.alloc(&b2, 50)) == cudaSuccess) e = tmp.alloc(&t, 7);
            if (e != cudaSuccess) {
                CHECK(e == cudaErrorMemoryAllocation);
                CHECK(fail_at >= 1 && fail_at <= 3);
                CHECK((fail_at == 1) == (a2 == a) && (fail_at <= 2) == (b2 == b));   // a failed alloc leaves its pointer untouched
            } else {
                CHECK(fail_at == 0 || fail_at > 3);
                CHECK(fresh.bytes() == 320 + 200 && tmp.bytes() == 56 && live(Dev) == 6);
                own.free(a);
                own.free(b);
                own.take(std::move(fresh));
                CHECK(fresh.bytes() == 0);
                a = a2;
                b = b2;
                ok = true;
            }
        }
        // the local sets are gone: on failure everything they held is freed and the handle's set is as it was
        if (ok) CHECK(own.bytes() == 320 + 200 + 3 && live(Dev) == 3 && g_live.count(a) && g_live.count(b) && g_live.count(c));
        else CHECK(own.bytes() == 80 + 80 + 3 && live(Dev) == 3 && g_live.count(a) && g_live.count(b) && g_live.count(c));
        own.free(c);
        CHECK(own.bytes() == (ok ? 520u : 160u) && live(Dev) == 2 && !g_live.count(c));
        own.free(nullptr);   // nothing
        CHECK(live(Dev) == 2);
    }
    CHECK(live(Dev) == 0 && live(Host) == 0);
    return 0;
}

// grow-only scratch: the allocation calls of the scenario are numbered from 1 (the first two may fail); `pinned` picks the kind
int dm_regrow(long long fail_at, int pinned) {
    dm_reset(fail_at);
    const Kind k = pinned ? Host : Dev;
    {
        MemSet s(pinned ? MemSet::Pinned : MemSet::Device);
        float* p = nullptr;
        size_t cap = 0;
        // call 1: from empty, at the floor
        cudaError_t e = s.regrow(&p, &cap, 10, 1024);
        if (fail_at == 1) {
            CHECK(e == cudaErrorMemoryAllocation && !p && cap == 0 && s.bytes() == 0 && live(k) == 0);
            g_fail_at = 0;
            e = s.regrow(&p, &cap, 10, 1024);   // retryable
        }
        CHECK(e == cudaSuccess && p && cap == 1024 && s.bytes() == 4096 && live(k) == 1);
        // no call: need <= cap keeps the block
        float* const p1 = p;
        const long long calls = g_allocs;
        CHECK(s.regrow(&p, &cap, 1024, 1024) == cudaSuccess && p == p1 && cap == 1024 && g_allocs == calls);
        CHECK(s.regrow(&p, &cap, 0) == cudaSuccess && p == p1 && cap == 1024);
        // the next growing call: the old block is freed before the new one is allocated; need above the floor is taken as it is
        const long long seq0 = g_seq;
        e = s.regrow(&p, &cap, 3000, 1024);
        CHECK(g_last_free_seq > seq0);
        if (e != cudaSuccess) {
            CHECK(fail_at == calls + 1 && !p && cap == 0 && s.bytes() == 0 && live(k) == 0);
            g_fail_at = 0;
            e = s.regrow(&p, &cap, 3000, 1024);
        } else {
            CHECK(g_last_alloc_seq > g_last_free_seq);
        }
        CHECK(e == cudaSuccess && p && cap == 3000 && s.bytes() == 12000 && live(k) == 1);
        // exactly `need` without a floor
        g_fail_at = 0;
        CHECK(s.regrow(&p, &cap, 3001) == cudaSuccess && cap == 3001 && s.bytes() == 12004 && live(k) == 1);
        CHECK(live(pinned ? Dev : Host) == 0);
    }
    CHECK(live(Dev) == 0 && live(Host) == 0);
    return 0;
}

// memset_byte: applied to device blocks (cudaMemset) and pinned ones; a failed memset leaves nothing behind
int dm_memset() {
    dm_reset(0);
    {
        MemSet d, h(MemSet::Pinned);
        unsigned char *p = nullptr, *q = nullptr;
        CHECK(d.alloc(&p, 37, 0xAB) == cudaSuccess && h.alloc(&q, 19, 0x5C) == cudaSuccess);
        for (int i = 0; i < 37; ++i) CHECK(p[i] == 0xAB);
        for (int i = 0; i < 19; ++i) CHECK(q[i] == 0x5C);
        int* r = nullptr;
        CHECK(d.alloc(&r, 5, 0) == cudaSuccess);
        for (int i = 0; i < 5; ++i) CHECK(r[i] == 0);
        g_memset_fail = 1;
        int* const sentinel = reinterpret_cast<int*>(0x10);
        int* f = sentinel;
        CHECK(d.alloc(&f, 8, 0xFF) != cudaSuccess && f == sentinel && d.bytes() == 37 + 20 && live(Dev) == 2);
        g_memset_fail = 0;
    }
    CHECK(live(Dev) == 0 && live(Host) == 0);
    return 0;
}

// kinds and moves: pinned blocks go back through cudaFreeHost, device blocks through cudaFree (the stubs count any mix-up); a
// moved-from set frees nothing; move assignment frees what the target held; take joins two sets of one kind
int dm_kinds_and_moves() {
    dm_reset(0);
    {
        MemSet d, h(MemSet::Pinned);
        int* a = nullptr;
        double* b = nullptr;
        CHECK(d.alloc(&a, 4) == cudaSuccess && h.alloc(&b, 4) == cudaSuccess && live(Dev) == 1 && live(Host) == 1);
        {
            MemSet moved(std::move(h));
            CHECK(h.bytes() == 0 && moved.bytes() == 32);
            MemSet h2(MemSet::Pinned);
            double* c = nullptr;
            CHECK(h2.alloc(&c, 2) == cudaSuccess && live(Host) == 2);
            moved.take(std::move(h2));
            CHECK(moved.bytes() == 48 && h2.bytes() == 0 && live(Host) == 2);
            h.free(b);   // not in the moved-from set any more: nothing
            CHECK(live(Host) == 2);
        }
        CHECK(live(Host) == 0 && live(Dev) == 1);
        MemSet e;
        int* x = nullptr;
        CHECK(e.alloc(&x, 3) == cudaSuccess && live(Dev) == 2);
        e = std::move(d);   // x is freed, a now belongs to e
        CHECK(live(Dev) == 1 && g_live.count(a) && !g_live.count(x) && e.bytes() == 16 && d.bytes() == 0);
        e = MemSet();       // cleared by assignment
        CHECK(live(Dev) == 0 && e.bytes() == 0);
    }
    CHECK(live(Dev) == 0 && live(Host) == 0);
    return 0;
}
}  // extern "C"
