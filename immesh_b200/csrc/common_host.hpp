// immesh_b200 -- host-side helpers shared by the C-ABI translation units: error reporting, launch accounting
// and an optional CUDA-event profiler (per-kernel device time on the launching stream, used by bench.py for the
// roofline numbers; off by default so that timed runs carry no event overhead).
#pragma once
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/immesh_b200.h"
#include "dev_mem.hpp"

namespace immesh {
// a handle under construction: every return before release() hands it to its destroy function, which copes with a handle built
// only in part (its memory is held by MemSet members)
template <class H>
using Building = std::unique_ptr<H, int (*)(H*)>;

// true when `p` is page-locked host memory the device can read directly (allocated pinned, or registered): such an input is
// copied straight from the caller's buffer, without the staging memcpy
inline bool host_ptr_is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// H2D on the upload stream, overlapping earlier kernels, joined by `st` through `ev`; an unpinned source goes through `stage` if given
inline cudaError_t upload_async(void* dst, const void* src, size_t bytes, void* stage, cudaStream_t up, cudaEvent_t ev, cudaStream_t st) {
    if (stage && !host_ptr_is_pinned(src)) src = std::memcpy(stage, src, bytes);
    cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, up);
    if (e == cudaSuccess) e = cudaEventRecord(ev, up);
    return e == cudaSuccess ? cudaStreamWaitEvent(st, ev, 0) : e;
}

inline std::string& last_error_storage() {
    static thread_local std::string s;
    return s;
}
inline int im_fail(int code, const char* msg) {
    last_error_storage() = msg ? msg : "";
    return code;
}
// a failed allocation of a call's buffers (the sticky error cleared): IMMESH_E_CAPACITY when memory ran out, IMMESH_E_CUDA otherwise
inline int im_fail_alloc(cudaError_t e, const char* msg) {
    cudaGetLastError();
    return im_fail(e == cudaErrorMemoryAllocation ? IMMESH_E_CAPACITY : IMMESH_E_CUDA, msg);
}
inline int im_fail_cuda(cudaError_t e, const char* file, int line) {
    char buf[512];
    std::snprintf(buf, sizeof(buf), "CUDA error %d (%s) at %s:%d", (int)e, cudaGetErrorString(e), file, line);
    last_error_storage() = buf;
    return IMMESH_E_CUDA;
}

struct Profiler {
    bool enabled = false;
    long long launches = 0;
    struct Rec { const char* name; cudaEvent_t a, b; };
    std::vector<Rec> pending;
    std::vector<cudaEvent_t> pool;
    std::map<std::string, std::pair<double, long long>> totals;  // name -> (ms, launches)
    cudaEvent_t get_event() {
        if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
        cudaEvent_t e;
        cudaEventCreate(&e);
        return e;
    }
    void begin(const char* name, cudaStream_t st) {
        Rec r{name, get_event(), get_event()};
        cudaEventRecord(r.a, st);
        pending.push_back(r);
    }
    void end(cudaStream_t st) { cudaEventRecord(pending.back().b, st); }
    // optional timeline: start/end of every launch relative to a base event (diagnosis of the two-stream pipeline)
    bool timeline_on = false;
    cudaEvent_t base = nullptr;
    struct Span { const char* name; float t0, t1; };
    std::vector<Span> timeline;
    void start_timeline() {
        if (!base) cudaEventCreate(&base);
        cudaDeviceSynchronize();
        cudaEventRecord(base, 0);
        cudaEventSynchronize(base);
        timeline.clear();
        timeline_on = true;
    }
    void collect() {  // harvests every launch whose end event has completed; the others stay pending
        std::vector<Rec> keep;
        for (Rec& r : pending) {
            if (cudaEventQuery(r.b) == cudaErrorNotReady) { keep.push_back(r); continue; }
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
                auto& t = totals[r.name];
                t.first += ms;
                t.second += 1;
                if (timeline_on) {
                    Span sp{r.name, 0.f, 0.f};
                    cudaEventElapsedTime(&sp.t0, base, r.a);
                    cudaEventElapsedTime(&sp.t1, base, r.b);
                    timeline.push_back(sp);
                }
            }
            pool.push_back(r.a);
            pool.push_back(r.b);
        }
        pending.swap(keep);
        cudaGetLastError();
    }
};
Profiler& profiler();  // defined in misc_capi.cu
}  // namespace immesh

#define IM_CUDA(expr)                                                              \
    do {                                                                           \
        cudaError_t im_e_ = (expr);                                                \
        if (im_e_ != cudaSuccess) return immesh::im_fail_cuda(im_e_, __FILE__, __LINE__); \
    } while (0)

// ---- CUDA-graph replay of a fixed launch sequence.  The per-scan work is ~40 short kernels, so queueing them one by
// one is host-launch-bound.  The first pipelined call runs the host code path under stream capture, recording its launches
// into a graph; every later call replays that graph with ONE cudaGraphLaunch and runs no host code of the sequence.  Outside
// a capture (graph_ctx() null), IM_LAUNCH launches directly.
namespace immesh {
struct GraphCtx {
    cudaGraphExec_t exec = nullptr;
    cudaGraph_t graph = nullptr;
    long long kernels = 0;             // kernel launches recorded into the graph
    long long pdl_edges = 0;           // programmatic (IM_LAUNCH_PDL) edges of the captured graph
    unsigned sig = 0;                  // control-flow signature the graph was captured with
    cudaError_t err = cudaSuccess;
    long long captures = 0, replays = 0, failures = 0;
    void destroy() {
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
        exec = nullptr; graph = nullptr; kernels = 0; pdl_edges = 0;
    }
};
inline GraphCtx*& graph_ctx() {
    static thread_local GraphCtx* g = nullptr;
    return g;
}
// pdl: launch with programmatic stream serialization (Hopper programmatic dependent launch): the kernel may be scheduled while the
// previous kernel on `st` still runs, and must call pdl_wait() (pdl.cuh) before it touches global memory.  Only for a kernel that
// directly follows another kernel on the same stream; under stream capture the attribute becomes a programmatic graph edge.
template <typename... KArgs, typename... Args>
inline void im_launch(const char* name, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args&&... args) {
    Profiler& pr = profiler();
    pr.launches++;
    std::tuple<KArgs...> vals(std::forward<Args>(args)...);   // exactly the kernel's parameter types
    void* ptrs[sizeof...(KArgs) ? sizeof...(KArgs) : 1];
    {
        size_t k = 0;
        std::apply([&](auto&... v) { ((ptrs[k++] = (void*)&v), ...); }, vals);
    }
    GraphCtx* g = graph_ctx();
    if (pr.enabled) pr.begin(name, st);
    cudaError_t e;
    if (pdl) {
        cudaLaunchAttribute attr;
        attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr.val.programmaticStreamSerializationAllowed = 1;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
        cfg.attrs = &attr; cfg.numAttrs = 1;
        e = cudaLaunchKernelExC(&cfg, (const void*)kern, ptrs);
    } else {
        e = cudaLaunchKernel((const void*)kern, grid, block, ptrs, smem, st);
    }
    if (pr.enabled) pr.end(st);
    if (g) {   // capturing: the launch must have been recorded on a stream of the capture
        cudaStreamCaptureStatus status;
        cudaError_t e2 = cudaStreamGetCaptureInfo(st, &status);
        if (e == cudaSuccess && e2 == cudaSuccess && status == cudaStreamCaptureStatusActive) g->kernels++;
        else if (g->err == cudaSuccess) g->err = (e != cudaSuccess) ? e : (e2 != cudaSuccess ? e2 : cudaErrorUnknown);
    }
}
inline cudaError_t count_pdl_edges(GraphCtx& g) {
    size_t n = 0;
    cudaError_t e = cudaGraphGetEdges_v2(g.graph, nullptr, nullptr, nullptr, &n);
    if (e != cudaSuccess || n == 0) return e;
    std::vector<cudaGraphNode_t> from(n), to(n);
    std::vector<cudaGraphEdgeData> data(n);
    e = cudaGraphGetEdges_v2(g.graph, from.data(), to.data(), data.data(), &n);
    if (e != cudaSuccess) return e;
    g.pdl_edges = 0;
    for (size_t i = 0; i < n; ++i) g.pdl_edges += data[i].type == cudaGraphDependencyTypeProgrammatic;
    return cudaSuccess;
}
// The body's launches take every per-call value from device memory, so once captured the graph is replayed by a bare
// cudaGraphLaunch -- the body is not run again.  `sig` must cover everything that changes the sequence or its arguments
// (handle pointers, modes, iteration counts).
template <typename Body>
inline cudaError_t run_graphed_static(GraphCtx& g, unsigned sig, cudaStream_t st, Body&& body) {
    if (g.exec && g.sig != sig) g.destroy();
    if (!g.exec) {
        g.err = cudaSuccess;
        g.kernels = 0;
        graph_ctx() = &g;
        cudaError_t e = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
        if (e != cudaSuccess) { graph_ctx() = nullptr; return e; }
        body();
        graph_ctx() = nullptr;
        e = cudaStreamEndCapture(st, &g.graph);
        if (e == cudaSuccess && g.err != cudaSuccess) e = g.err;
        if (e == cudaSuccess) e = cudaGraphInstantiate(&g.exec, g.graph, 0);
        if (e == cudaSuccess) e = count_pdl_edges(g);
        if (e != cudaSuccess) { g.destroy(); cudaGetLastError(); g.failures++; return e; }
        g.sig = sig;
        g.captures++;
    } else {
        g.replays++;
        profiler().launches += g.kernels;   // launch accounting: every kernel of the graph runs
    }
    return cudaGraphLaunch(g.exec, st);
}
}  // namespace immesh

// an enable's start: work in flight uses the stage's buffers and the captured sequence changes, so drain and drop the graph first
template <class H, class Reset>
inline cudaError_t im_stage_reset(H* h, Reset&& reset) {
    const cudaError_t e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) return e;
    h->graph.destroy();
    reset();
    return cudaSuccess;
}

// kernel launch with accounting; wrap template kernels in parentheses: IM_LAUNCH((k<256>), grid, block, smem, stream, args...)
#define IM_LAUNCH(KERN, GRID, BLOCK, SMEM, STREAM, ...) immesh::im_launch(#KERN, KERN, dim3(GRID), dim3(BLOCK), (SMEM), (STREAM), false, ##__VA_ARGS__)
// the same, with programmatic dependent launch when PDL is true (see im_launch; KERN must call pdl_wait() first on every path)
#define IM_LAUNCH_PDL(PDL, KERN, GRID, BLOCK, SMEM, STREAM, ...) immesh::im_launch(#KERN, KERN, dim3(GRID), dim3(BLOCK), (SMEM), (STREAM), (bool)(PDL), ##__VA_ARGS__)
