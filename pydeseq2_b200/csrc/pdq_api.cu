// pdq_api.cu -- the C ABI declared in include/pydeseq2_b200.h (context, memory, host-buffer and
// device-resident entry points, NCCL gene-shard exchange).  Host code only; kernels live in
// pdq_kernels.cu, pdq_wide.cu, pdq_common.cu and pdq_padj.cu.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <condition_variable>
#include <functional>
#include <initializer_list>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "pdq_internal.h"
#include "pdq_host_linalg.h"
#include "pdq_padj.cuh"

using namespace pdq;

// --------------------------------------------------------------------------------------------- host worker threads
// A few persistent host threads for the two memory-bound host loops of the host-buffer path (content checksums, staging copies of
// pageable buffers).  Workers SLEEP between jobs (condition variable): with one process per GPU, eight ranks share the host, and
// spinning runtimes (OpenMP's default wait policy) made eight ranks slower than one.  Threads per process: the host's hardware
// threads divided by the ranks on it (LOCAL_WORLD_SIZE), at most 32; PDQ_HOST_THREADS overrides.
class HostPool {
public:
    static HostPool& get() {
        static HostPool p;
        return p;
    }
    int size() const { return n_; }
    // f(t, nt) for t = 0 .. nt-1, the caller runs t = 0
    void run(int nt, const std::function<void(int, int)>& f) {
        if (nt > n_) nt = n_;
        if (nt <= 1) {
            f(0, 1);
            return;
        }
        {
            std::unique_lock<std::mutex> lk(m_);
            job_ = &f;
            nt_ = nt;
            pending_ = nt - 1;
            ++gen_;
        }
        cv_.notify_all();
        f(0, nt);
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [&] { return pending_ == 0; });
        job_ = nullptr;
    }

private:
    HostPool() {
        int hw = (int)std::thread::hardware_concurrency();
        if (hw < 1) hw = 1;
        int ranks = 1;
        if (const char* e = getenv("LOCAL_WORLD_SIZE")) ranks = atoi(e) > 0 ? atoi(e) : 1;
        n_ = hw / ranks;
        if (n_ > 32) n_ = 32;
        if (const char* e = getenv("PDQ_HOST_THREADS")) n_ = atoi(e);
        if (n_ < 1) n_ = 1;
        for (int t = 1; t < n_; ++t) th_.emplace_back([this, t] { loop(t); });
    }
    ~HostPool() {
        {
            std::unique_lock<std::mutex> lk(m_);
            stop_ = true;
            ++gen_;
        }
        cv_.notify_all();
        for (auto& t : th_) t.join();
    }
    void loop(int t) {
        uint64_t seen = 0;
        for (;;) {
            const std::function<void(int, int)>* job = nullptr;
            int nt = 0;
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_.wait(lk, [&] { return gen_ != seen; });
                seen = gen_;
                if (stop_) return;
                if (t >= nt_) continue;  // this job uses fewer threads
                job = job_;
                nt = nt_;
            }
            (*job)(t, nt);
            std::unique_lock<std::mutex> lk(m_);
            if (--pending_ == 0) done_.notify_one();
        }
    }
    std::vector<std::thread> th_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    const std::function<void(int, int)>* job_ = nullptr;
    int n_ = 1, nt_ = 0, pending_ = 0;
    uint64_t gen_ = 0;
    bool stop_ = false;
};

// --------------------------------------------------------------------------------------------- NCCL (dlopen)
// NCCL is resolved at run time so that the library loads on boxes without it and never clashes with
// the copy a host application (e.g. torch) already mapped: the soname lookup returns that same copy.
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static const int kNcclFloat64 = 8;  // ncclDataType_t::ncclFloat64 (stable across NCCL 2.x)

enum { kBufCounts, kBufA, kBufB, kBufC, kBufD, kBufE, kBufF, kBufG, kBufStatus, kBufMisc, kBufKeep, kBufRes, kBufPadj, kBufCooks, kNumBufs };

struct DesignCacheEntry {
    pdq_design* d = nullptr;
    std::vector<double> X, sf;
    bool offsets = false;  // `sf` holds log size factors given by the caller (apeGLM offsets)
    uint64_t stamp = 0;
};

struct pdq_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaDeviceProp prop{};
    int lanes_override = 0;
    int64_t launches = 0;
    std::string err;
    void* buf[kNumBufs] = {};
    size_t cap[kNumBufs] = {};
    // design packs of the host-buffer entry points, keyed on the bytes of X and the size factors (small LRU)
    std::vector<DesignCacheEntry> dcache;
    uint64_t dcache_clock = 0;
    // page-locked staging ring for pageable host buffers (numpy arrays are pageable)
    void* stage[2] = {nullptr, nullptr};
    cudaEvent_t stage_ev[2] = {nullptr, nullptr};
    bool stage_busy[2] = {false, false};
    int staging = 1;  // PDQ_STAGING=0 disables (plain cudaMemcpyAsync from pageable memory)
    int* tickets = nullptr;  // device ints for the persistent kernels' tile counters (4 per stream slot), then the control words of
                             // the fused MAP -> LFC launch (launch_map_irls); zeroed once, here
    unsigned* tile_done = nullptr;  // per-tile hand-off words of launch_map_irls (zeroed when allocated)
    size_t tile_cap = 0;
    unsigned long long* tail_err_host = nullptr;  // mapped page-locked word: non-zero after a tile wait of launch_map_irls gave up
    unsigned long long* tail_err_dev = nullptr;
    void* grid_scratch = nullptr;  // accumulators of the grid-wide trend fit
    cudaStream_t pstream[2] = {nullptr, nullptr};  // gene-block pipeline of the host-buffer entry points
    cudaEvent_t pfork = nullptr, pjoin[2] = {nullptr, nullptr};
    cudaStream_t cstream = nullptr;  // side copies of the resident pass (pdq_memcpy_d2h_side): a branch that rejoins `stream`
    cudaEvent_t cfork = nullptr, cjoin = nullptr;
    bool side_pending = false;       // a side copy was enqueued since the last pdq_side_join
    int pipeline = 4;        // gene blocks per pipelined call; PDQ_PIPELINE=0 disables
    int debug = 0;           // PDQ_DEBUG_* test hooks
    int wide = 0;            // designs of up to PDQ_MAX_P_WIDE columns (pdq_set_wide_designs)
    int wide_shrink = 0;     // apeGLM shrinkage of those designs (pdq_set_wide_shrink)
    int large = 0;           // designs of up to PDQ_MAX_P_LARGE columns, with `wide` on as well (pdq_set_large_designs)
    int large_shrink = 0;    // apeGLM shrinkage of those, with `wide_shrink` and `large` on as well (pdq_set_large_shrink)
    int64_t launches_at_capture = 0;
    int64_t buf_epoch = 0;   // bumped whenever ensure() re-allocates a context-owned buffer (captured graphs hold those pointers)
    NcclApi nccl;
    ncclComm_t comm = nullptr;
    int world = 1, rank = 0;
    // content-addressed residency of the (N, G) buffers of the host-buffer entry points (see "residency" below)
    struct ResEntry {
        uint64_t h[2];
        size_t bytes;
        void* dptr;
        uint64_t stamp;   // LRU clock
        uint64_t call;    // id of the last call that used the entry (entries of the running call are never evicted)
        int pending;      // >= 0: output whose device-side hash lands in hash_host[2 * pending] after the call's final sync
        int state;        // 0 spare allocation, 1 being filled by the running call, 2 valid
    };
    std::vector<ResEntry*> res;  // heap objects: a slot handed to a call stays valid when other entries are evicted
    size_t res_bytes = 0, res_cap = 0;
    uint64_t res_clock = 0, res_call = 0;
    int residency = 1;           // PDQ_RESIDENCY=0 disables
    uint64_t* hash_dev = nullptr;   // 2 x 8 slots
    uint64_t* hash_host = nullptr;  // page-locked mirror
    int hash_pending = 0;
    int64_t res_hits = 0, res_misses = 0;
    int64_t res_hit_bytes = 0;
};

struct pdq_design {
    DesignDev d;
};

static int fail(pdq_ctx* c, int code, const char* fmt, ...) {
    if (c) {
        char tmp[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(tmp, sizeof tmp, fmt, ap);
        va_end(ap);
        c->err = tmp;
    }
    return code;
}

#define CU(c, call)                                                                                  \
    do {                                                                                             \
        cudaError_t e__ = (call);                                                                    \
        if (e__ != cudaSuccess)                                                                      \
            return fail(c, PDQ_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

static int ensure(pdq_ctx* c, int which, size_t bytes, void** out) {
    if (bytes > c->cap[which]) {
        if (c->buf[which]) {
            CU(c, cudaFree(c->buf[which]));
            ++c->buf_epoch;
        }
        c->buf[which] = nullptr;
        c->cap[which] = 0;
        const size_t want = bytes + bytes / 8 + 256;
        CU(c, cudaMalloc(&c->buf[which], want));
        c->cap[which] = want;
    }
    *out = c->buf[which];
    return 0;
}

static int pick_lgT(const pdq_ctx* c, int G, int N) {
    int T;
    if (c->lanes_override) {
        T = c->lanes_override;
    } else {
        // fill ~1024 resident threads per SM: T = smallest power of two with G*T >= SMs*1024, capped by 32 -- but never
        // fewer than 8 lanes: a warp then owns 4 adjacent genes = one full 32-byte sector per sample row, and its tile
        // (4 genes x N samples x 16 B for counts + means) stays small enough for the resident warps of an SM to keep
        // their tiles in L2 across evaluations.  The SM count comes from the device (132 on H100); scripts/lanes_sweep.sh
        // times the alternatives.
        const double want = (double)c->prop.multiProcessorCount * 1024.0 / (double)(G > 0 ? G : 1);
        T = 8;
        while (T < 32 && (double)T < want) T <<= 1;
    }
    while (T > 1 && T > N) T >>= 1;  // never more lanes than samples
    int lg = 0;
    while ((1 << lg) < T) ++lg;
    return lg;
}

static LaunchCfg cfg(const pdq_ctx* c, int G, int N) { return LaunchCfg{c->stream, pick_lgT(c, G, N), c->prop.multiProcessorCount, c->tickets, c->debug}; }

// --------------------------------------------------------------------------------------------- context
extern "C" const char* pdq_version(void) { return "pydeseq2_b200 0.1.0 (sm_90a)"; }

extern "C" int pdq_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

extern "C" int pdq_ctx_create(int device, pdq_ctx** out) {
    if (!out) return PDQ_ERR_INVALID;
    *out = nullptr;
    int n = pdq_device_count();
    if (n <= 0 || device < 0 || device >= n) return PDQ_ERR_NO_DEVICE;
    pdq_ctx* c = new pdq_ctx();
    c->device = device;
    if (cudaSetDevice(device) != cudaSuccess || cudaGetDeviceProperties(&c->prop, device) != cudaSuccess) {
        delete c;
        return PDQ_ERR_NO_DEVICE;
    }
    if (c->prop.major != 9 || c->prop.minor != 0) {  // the fatbin holds sm_90a SASS only, which loads on compute capability 9.0 alone
        delete c;
        return PDQ_ERR_NO_DEVICE;
    }
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete c;
        return PDQ_ERR_CUDA;
    }
    for (auto& e : c->ev)
        if (cudaEventCreate(&e) != cudaSuccess) {
            delete c;
            return PDQ_ERR_CUDA;
        }
    if (const char* s = getenv("PDQ_STAGING")) c->staging = atoi(s);
    if (const char* s = getenv("PDQ_PIPELINE")) c->pipeline = atoi(s);
    if (const char* s = getenv("PDQ_RESIDENCY")) c->residency = atoi(s);
    c->res_cap = c->prop.totalGlobalMem / 4;
    if (c->res_cap > ((size_t)16 << 30)) c->res_cap = (size_t)16 << 30;
    if (const char* s = getenv("PDQ_RESIDENCY_BYTES")) c->res_cap = (size_t)atoll(s);
    if (cudaMalloc((void**)&c->tickets, 128) != cudaSuccess || cudaMemsetAsync(c->tickets, 0, 128, c->stream) != cudaSuccess || cudaMalloc(&c->grid_scratch, kGridScratchBytes) != cudaSuccess || cudaStreamCreateWithFlags(&c->pstream[0], cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->pstream[1], cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->pfork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->pjoin[0], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->pjoin[1], cudaEventDisableTiming) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->cstream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->cfork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->cjoin, cudaEventDisableTiming) != cudaSuccess) {
        delete c;
        return PDQ_ERR_CUDA;
    }
    *out = c;
    return PDQ_OK;
}

extern "C" void pdq_ctx_destroy(pdq_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->comm && c->nccl.CommDestroy) c->nccl.CommDestroy(c->comm);
    for (auto& e : c->dcache) pdq_design_destroy(c, e.d);
    c->dcache.clear();
    for (auto& b : c->buf)
        if (b) cudaFree(b);
    for (auto* e : c->res) {
        if (e->dptr) cudaFree(e->dptr);
        delete e;
    }
    if (c->hash_dev) cudaFree(c->hash_dev);
    if (c->hash_host) cudaFreeHost(c->hash_host);
    if (c->tickets) cudaFree(c->tickets);
    if (c->tile_done) cudaFree(c->tile_done);
    if (c->tail_err_host) cudaFreeHost(c->tail_err_host);
    if (c->grid_scratch) cudaFree(c->grid_scratch);
    for (auto& st : c->pstream)
        if (st) cudaStreamDestroy(st);
    if (c->pfork) cudaEventDestroy(c->pfork);
    for (auto& ev : c->pjoin)
        if (ev) cudaEventDestroy(ev);
    if (c->cstream) cudaStreamDestroy(c->cstream);
    if (c->cfork) cudaEventDestroy(c->cfork);
    if (c->cjoin) cudaEventDestroy(c->cjoin);
    for (int i = 0; i < 2; ++i) {
        if (c->stage[i]) cudaFreeHost(c->stage[i]);
        if (c->stage_ev[i]) cudaEventDestroy(c->stage_ev[i]);
    }
    for (auto& e : c->ev)
        if (e) cudaEventDestroy(e);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

extern "C" const char* pdq_last_error(const pdq_ctx* c) { return c ? c->err.c_str() : "null context"; }

extern "C" int pdq_device_info(const pdq_ctx* c, char* name, size_t name_len, int* sm_count, size_t* mem_bytes) {
    if (!c) return PDQ_ERR_INVALID;
    if (name && name_len) {
        strncpy(name, c->prop.name, name_len - 1);
        name[name_len - 1] = 0;
    }
    if (sm_count) *sm_count = c->prop.multiProcessorCount;
    if (mem_bytes) *mem_bytes = c->prop.totalGlobalMem;
    return PDQ_OK;
}

extern "C" int pdq_set_lanes_per_gene(pdq_ctx* c, int lanes) {
    if (!c) return PDQ_ERR_INVALID;
    if (lanes != 0 && (lanes < 1 || lanes > 32 || (lanes & (lanes - 1)))) return fail(c, PDQ_ERR_INVALID, "lanes per gene must be 0 or a power of two <= 32");
    c->lanes_override = lanes;
    return PDQ_OK;
}

extern "C" int pdq_set_debug_flags(pdq_ctx* c, int flags) {
    if (!c) return PDQ_ERR_INVALID;
    c->debug = flags;
    return PDQ_OK;
}

extern "C" int pdq_set_wide_designs(pdq_ctx* c, int on) {
    if (!c) return PDQ_ERR_INVALID;
    c->wide = on != 0;
    return PDQ_OK;
}

extern "C" int pdq_set_wide_shrink(pdq_ctx* c, int on) {
    if (!c) return PDQ_ERR_INVALID;
    c->wide_shrink = on != 0;
    return PDQ_OK;
}

extern "C" int pdq_set_large_designs(pdq_ctx* c, int on) {
    if (!c) return PDQ_ERR_INVALID;
    c->large = on != 0;
    return PDQ_OK;
}

extern "C" int pdq_set_large_shrink(pdq_ctx* c, int on) {
    if (!c) return PDQ_ERR_INVALID;
    c->large_shrink = on != 0;
    return PDQ_OK;
}

extern "C" int pdq_design_pinv(const double* X, int N, int p, double* pinv_out, int* full_rank_out) {
    if (!X || !pinv_out || !full_rank_out || N <= 0 || p < 1 || p > PDQ_MAX_P_WIDE) return PDQ_ERR_INVALID;
    design_linear_algebra(X, N, p, pinv_out, full_rank_out);
    return PDQ_OK;
}

extern "C" int pdq_design_pinv_large(const double* X, int N, int p, double* pinv_out, int* full_rank_out) {
    if (!X || !pinv_out || !full_rank_out || N <= 0 || p < 1 || p > PDQ_MAX_P_LARGE) return PDQ_ERR_INVALID;
    design_linear_algebra(X, N, p, pinv_out, full_rank_out);
    return PDQ_OK;
}

extern "C" int64_t pdq_launch_count(const pdq_ctx* c) { return c ? c->launches : 0; }
extern "C" int64_t pdq_buffer_epoch(const pdq_ctx* c) { return c ? c->buf_epoch : 0; }

extern "C" int pdq_malloc(pdq_ctx* c, size_t bytes, void** dptr) {
    if (!c || !dptr) return PDQ_ERR_INVALID;
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaMalloc(dptr, bytes ? bytes : 1));
    return PDQ_OK;
}
extern "C" int pdq_free(pdq_ctx* c, void* dptr) {
    if (!c) return PDQ_ERR_INVALID;
    if (dptr) CU(c, cudaFree(dptr));
    return PDQ_OK;
}
extern "C" int pdq_host_alloc(pdq_ctx* c, size_t bytes, void** hptr) {
    if (!c || !hptr) return PDQ_ERR_INVALID;
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaHostAlloc(hptr, bytes ? bytes : 1, cudaHostAllocDefault));
    return PDQ_OK;
}
extern "C" int pdq_host_free(pdq_ctx* c, void* hptr) {
    if (!c) return PDQ_ERR_INVALID;
    if (hptr) CU(c, cudaFreeHost(hptr));
    return PDQ_OK;
}
extern "C" int pdq_memcpy_h2d(pdq_ctx* c, void* dst, const void* src, size_t bytes) {
    if (!c) return PDQ_ERR_INVALID;
    CU(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->stream));
    return PDQ_OK;
}
extern "C" int pdq_memcpy_d2h(pdq_ctx* c, void* dst, const void* src, size_t bytes) {
    if (!c) return PDQ_ERR_INVALID;
    CU(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
    return PDQ_OK;
}
extern "C" int pdq_memcpy_d2h_strided(pdq_ctx* c, void* dst, const void* src, size_t elem_bytes, size_t src_stride, size_t count) {
    if (!c || elem_bytes == 0 || src_stride < elem_bytes) return PDQ_ERR_INVALID;
    if (count) CU(c, cudaMemcpy2DAsync(dst, elem_bytes, src, src_stride, elem_bytes, count, cudaMemcpyDeviceToHost, c->stream));
    return PDQ_OK;
}
// A device-to-host copy on a branch of the context's stream: it starts behind the work enqueued so far and runs while the work
// enqueued after it does; pdq_side_join puts the stream behind every side copy since the last join.  Under stream capture the
// pair becomes a branch of the graph.
extern "C" int pdq_memcpy_d2h_side(pdq_ctx* c, void* dst, const void* src, size_t bytes) {
    if (!c) return PDQ_ERR_INVALID;
    CU(c, cudaEventRecord(c->cfork, c->stream));
    CU(c, cudaStreamWaitEvent(c->cstream, c->cfork, 0));
    CU(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->cstream));
    c->side_pending = true;
    return PDQ_OK;
}
extern "C" int pdq_side_join(pdq_ctx* c) {
    if (!c) return PDQ_ERR_INVALID;
    if (!c->side_pending) return PDQ_OK;  // nothing to join (and under capture the side stream may not be part of the graph)
    c->side_pending = false;
    CU(c, cudaEventRecord(c->cjoin, c->cstream));
    CU(c, cudaStreamWaitEvent(c->stream, c->cjoin, 0));
    return PDQ_OK;
}
extern "C" int pdq_memcpy_d2d(pdq_ctx* c, void* dst, const void* src, size_t bytes) {
    if (!c) return PDQ_ERR_INVALID;
    CU(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, c->stream));
    return PDQ_OK;
}
extern "C" int pdq_memset(pdq_ctx* c, void* dst, int value, size_t bytes) {
    if (!c) return PDQ_ERR_INVALID;
    CU(c, cudaMemsetAsync(dst, value, bytes, c->stream));
    return PDQ_OK;
}
extern "C" int pdq_sync(pdq_ctx* c) {
    if (!c) return PDQ_ERR_INVALID;
    CU(c, cudaStreamSynchronize(c->stream));
    return PDQ_OK;
}
extern "C" int pdq_event_record(pdq_ctx* c, int slot) {
    if (!c || slot < 0 || slot >= 4) return PDQ_ERR_INVALID;
    CU(c, cudaEventRecord(c->ev[slot], c->stream));
    return PDQ_OK;
}
extern "C" int pdq_event_elapsed_ms(pdq_ctx* c, int a, int b, float* ms) {
    if (!c || !ms || a < 0 || a >= 4 || b < 0 || b >= 4) return PDQ_ERR_INVALID;
    CU(c, cudaEventSynchronize(c->ev[b]));
    CU(c, cudaEventElapsedTime(ms, c->ev[a], c->ev[b]));
    return PDQ_OK;
}

#define CHECK_CTX(c) \
    if (!(c)) return PDQ_ERR_INVALID; \
    CU(c, cudaSetDevice((c)->device))

// --------------------------------------------------------------------------------------------- CUDA graphs
struct pdq_graph {
    cudaGraphExec_t exec = nullptr;
    int64_t kernels = 0;  // kernel nodes, added to the launch counter on every replay
};

extern "C" int pdq_capture_begin(pdq_ctx* c) {
    CHECK_CTX(c);
    c->launches_at_capture = c->launches;
    // relaxed: host-side CUDA calls that are not stream work (attribute / occupancy queries) stay legal while capturing
    CU(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeRelaxed));
    return PDQ_OK;
}

extern "C" int pdq_capture_end(pdq_ctx* c, pdq_graph** out) {
    CHECK_CTX(c);
    if (!out) return PDQ_ERR_INVALID;
    cudaGraph_t graph = nullptr;
    CU(c, cudaStreamEndCapture(c->stream, &graph));
    pdq_graph* g = new pdq_graph();
    g->kernels = c->launches - c->launches_at_capture;  // counted by the launchers while recording
    c->launches = c->launches_at_capture;               // recorded, not executed
    cudaError_t e = cudaGraphInstantiate(&g->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) {
        delete g;
        return fail(c, PDQ_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
    }
    *out = g;
    return PDQ_OK;
}

extern "C" int pdq_graph_launch(pdq_ctx* c, pdq_graph* g) {
    CHECK_CTX(c);
    if (!g || !g->exec) return PDQ_ERR_INVALID;
    CU(c, cudaGraphLaunch(g->exec, c->stream));
    c->launches += g->kernels;
    return PDQ_OK;
}

extern "C" void pdq_graph_destroy(pdq_ctx* c, pdq_graph* g) {
    if (!g) return;
    if (c) cudaSetDevice(c->device);
    if (g->exec) cudaGraphExecDestroy(g->exec);
    delete g;
}

// --------------------------------------------------------------------------------------------- design pack
// the widest design the context fits: PDQ_MAX_P, PDQ_MAX_P_WIDE after pdq_set_wide_designs(ctx, 1), PDQ_MAX_P_LARGE with large on too
static int max_p(const pdq_ctx* c) { return !c->wide ? PDQ_MAX_P : (c->large ? PDQ_MAX_P_LARGE : PDQ_MAX_P_WIDE); }

// Whether the context takes a design of p columns, for a fit or (`shrink`) for apeGLM shrinkage: up to max_p(c) columns, and for
// shrinkage of more than PDQ_MAX_P columns pdq_set_wide_shrink on top, of more than PDQ_MAX_P_WIDE pdq_set_large_shrink too.
// PDQ_OK, or the refusal the opt-ins call for (PDQ_ERR_UNSUPPORTED, behind `prefix`); p < 1 is refused as pdq_design_create does.
static int design_width(pdq_ctx* c, int p, bool shrink = false, const char* prefix = "") {
    if (p < 1) return fail(c, PDQ_ERR_INVALID, "pdq_design_create: bad arguments");
    auto no_shrink = [&](int q) {
        return fail(c, PDQ_ERR_UNSUPPORTED, "lfc_shrink: apeGLM shrinkage of designs with more than %d columns is not implemented", q);
    };
    if (shrink && p > PDQ_MAX_P && !c->wide_shrink) return no_shrink(PDQ_MAX_P);
    if (p > max_p(c))
        return fail(c, PDQ_ERR_UNSUPPORTED, "%sdesign has %d columns; %s p <= %d", prefix, p,
                    c->wide ? "wide designs support" : "this build supports", max_p(c));
    if (shrink && p > PDQ_MAX_P_WIDE && !c->large_shrink) return no_shrink(PDQ_MAX_P_WIDE);
    return PDQ_OK;
}

static int design_create(pdq_ctx* c, const double* X, const double* sf, bool offsets, int N, int p, pdq_design** out) {
    if (!c || !X || !out || N <= 0 || p < 1) return fail(c, PDQ_ERR_INVALID, "pdq_design_create: bad arguments");
    if (int e = design_width(c, p)) return e;
    CU(c, cudaSetDevice(c->device));
    pdq_design* d = new pdq_design();  // value-initialised: every device pointer starts null
    DesignDev& dd = d->d;
    dd.N = N;
    dd.p = p;
    dd.RS = design_row_stride(p);
    std::vector<double> pack;
    dd.s_mean_inv = design_pack(X, sf, offsets, N, p, pack);
    // Staging limit: a pack of up to 40 KB leaves room for four blocks per SM next to the math table and the per-gene tables of
    // the two heavy kernels; larger packs (N > ~1 280 at p = 2, ~850 at p = 3) are read from global memory, where they live in
    // L1 / L2 (every warp walks the same rows), so the number of samples is not bounded by shared memory.
    const size_t pack_bytes = pack.size() * 8;
    size_t stage_max = 40 * 1024;
    if (const char* e = getenv("PDQ_STAGE_MAX_BYTES")) stage_max = (size_t)atoll(e);  // tuning hook
    dd.staged = pack_bytes <= stage_max && pack_bytes + 16 <= kMaxDynSmem / 2;
    dd.smem_bytes = (dd.staged ? pack_bytes : 0) + 16;
    std::vector<double> pinv((size_t)p * p);
    design_linear_algebra(X, N, p, pinv.data(), &dd.full_rank);
    auto bail = [&](const char* what) {
        pdq_design_destroy(c, d);
        return fail(c, PDQ_ERR_CUDA, "%s failed", what);
    };
    if (p <= PDQ_MAX_P) {
        memcpy(dd.pinv, pinv.data(), pinv.size() * 8);
    } else if (cudaMalloc((void**)&dd.pinv_dev, pinv.size() * 8) != cudaSuccess ||
               cudaMemcpy(dd.pinv_dev, pinv.data(), pinv.size() * 8, cudaMemcpyHostToDevice) != cudaSuccess ||
               cudaMalloc((void**)&dd.wald_dev, ((size_t)p * (p + 1) / 2 + 1 + p) * 8) != cudaSuccess) {
        return bail("cudaMalloc/cudaMemcpy(pseudo-inverse)");
    }
    if (p > PDQ_MAX_P_WIDE)
        if (const char* e = getenv("PDQ_LARGE_WARPS")) dd.warps = atoi(e);  // tuning hook (A/B runs): 2, 4 or 8 warps per gene
    dd.few_rows = design_distinct_rows(X, N, p, 16) <= 16;
    if (const char* e = getenv("PDQ_IRLS_MEMO")) dd.few_rows = dd.few_rows && atoi(e) != 0;  // tuning hook (A/B runs)
    const std::vector<int> plan = design_cell_plan(X, N, p);
    dd.n_cells = plan[0];
    dd.plan_len = (int)plan.size();
    dd.n_in_cells = dd.plan_len - (2 + dd.n_cells + 1);
    if (cudaMalloc((void**)&dd.cell_plan, plan.size() * sizeof(int)) != cudaSuccess ||
        cudaMemcpy(dd.cell_plan, plan.data(), plan.size() * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess)
        return bail("cudaMalloc/cudaMemcpy(cell plan)");
    if (cudaMalloc((void**)&dd.pack, pack.size() * 8) != cudaSuccess) return bail("cudaMalloc(design pack)");
    // synchronous copy: `pack` is a temporary
    if (cudaMemcpy(dd.pack, pack.data(), pack.size() * 8, cudaMemcpyHostToDevice) != cudaSuccess) return bail("cudaMemcpy(design pack)");
    *out = d;
    return PDQ_OK;
}

extern "C" int pdq_design_create(pdq_ctx* c, const double* X, const double* sf, int N, int p, pdq_design** out) {
    return design_create(c, X, sf, false, N, p, out);
}

extern "C" void pdq_design_destroy(pdq_ctx* c, pdq_design* d) {
    if (!d) return;
    if (c) cudaSetDevice(c->device);
    if (d->d.pack) cudaFree(d->d.pack);
    if (d->d.cell_plan) cudaFree(d->d.cell_plan);
    if (d->d.pinv_dev) cudaFree(d->d.pinv_dev);
    if (d->d.wald_dev) cudaFree(d->d.wald_dev);
    delete d;
}

// design cache for the host-buffer entry points: deseq2() passes the same X (and size factors) to every call
static int cached_design(pdq_ctx* c, const double* X, const double* sf, int N, int p, pdq_design** out, bool offsets = false) {
    // a deseq2() pass alternates between three packs -- (X, sf), (X, no sf), (ones, sf) -- so a one-entry cache would
    // rebuild (SVD, cell plan, two cudaMallocs, two synchronous copies) on almost every call: keep the last few
    // a cached wide pack is refused again once the opt-in is off (entry points whose later checks rank below it ran it already)
    if (int e = design_width(c, p)) return e;
    const size_t nx = (size_t)N * p;
    for (size_t i = 0; i < c->dcache.size(); ++i) {
        DesignCacheEntry& e = c->dcache[i];
        if (e.d->d.N == N && e.d->d.p == p && e.X.size() == nx && memcmp(e.X.data(), X, nx * 8) == 0 &&
            ((sf == nullptr) == e.sf.empty()) && e.offsets == offsets && (!sf || memcmp(e.sf.data(), sf, (size_t)N * 8) == 0)) {
            e.stamp = ++c->dcache_clock;
            *out = e.d;
            return PDQ_OK;
        }
    }
    pdq_design* d = nullptr;
    if (int e = design_create(c, X, sf, offsets, N, p, &d)) return e;
    if (c->dcache.size() >= 4) {  // evict the least recently used pack
        size_t lru = 0;
        for (size_t i = 1; i < c->dcache.size(); ++i)
            if (c->dcache[i].stamp < c->dcache[lru].stamp) lru = i;
        pdq_design_destroy(c, c->dcache[lru].d);
        c->dcache.erase(c->dcache.begin() + lru);
    }
    DesignCacheEntry e;
    e.d = d;
    e.X.assign(X, X + nx);
    if (sf) e.sf.assign(sf, sf + N);
    e.offsets = offsets;
    e.stamp = ++c->dcache_clock;
    c->dcache.push_back(std::move(e));
    *out = d;
    return PDQ_OK;
}

// --------------------------------------------------------------------------------------------- device-resident ops
static int done(pdq_ctx* c, int rc, const char* what) {
    if (rc < 0) {
        if (rc == PDQ_ERR_UNSUPPORTED)
            return fail(c, rc, "%s: unsupported design (p=%d..%d, shared-memory stage <= %zu bytes)", what, 1, max_p(c), kMaxDynSmem);
        return fail(c, rc, "%s: kernel launch failed: %s", what, cudaGetErrorString(cudaGetLastError()));
    }
    c->launches += rc;
    return PDQ_OK;
}

// ---- operations: the checks and the launch behind both forms of an entry point
// An operation's semantic checks (those beyond null pointers and sizes) run before anything is staged, so that a refused call
// leaves the residency cache and the context's buffers as they were.  The device form launches once; the host-buffer form once
// per gene block, passing the block's slice of the per-gene scratch.
static int check_alt(pdq_ctx* c, int alt, const char* refusal) {
    return alt < 0 || alt > 4 ? fail(c, PDQ_ERR_INVALID, "%s", refusal) : PDQ_OK;
}

static int check_prior(pdq_ctx* c, int prior_reg, const double* prior_var_dev, double prior_disp_var) {
    return prior_reg && !prior_var_dev && !(prior_disp_var > 0.0) ? fail(c, PDQ_ERR_INVALID, "alpha_mle: prior_reg needs prior_disp_var > 0") : PDQ_OK;
}

static int check_not_square(pdq_ctx* c, int N, int p) {
    return N == p ? fail(c, PDQ_ERR_INVALID, "The number of samples and the number of design variables are equal") : PDQ_OK;
}

static int check_shrink(pdq_ctx* c, int p, int shrink_index, double prior_no_shrink_scale, double prior_scale) {
    const bool bad = shrink_index < 0 || shrink_index >= p || !(prior_no_shrink_scale > 0.0) || !(prior_scale > 0.0);
    return bad ? fail(c, PDQ_ERR_INVALID, "pdq_lfc_shrink_dev: bad arguments") : PDQ_OK;
}

// The fused launches (MAP -> LFC hand-off, moments fold) pay where a warp works on few tiles per launch; above 12 tiles per
// resident warp of the search the stages run as separate launches
static bool many_tiles(const LaunchCfg& lc, int G) {
    const int gpw = 32 >> lc.lgT;
    return (int64_t)(G + gpw - 1) / gpw > (int64_t)12 * 12 * lc.sm_count;
}

// `status`: per-gene scratch of G ints, nullptr for the context's
static int irls_op(pdq_ctx* c, const LaunchCfg& lc, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* disp,
                   const IrlsHost& h, double* beta, double* mu, double* hat, int64_t ld_out, double* conv, int* status, int* n_fallback,
                   const WaldHost* w = nullptr) {
    void* st = status;
    if (!st)
        if (int e = ensure(c, kBufStatus, (size_t)G * sizeof(int), &st)) return e;
    return done(c, launch_irls(lc, d, counts, ld, G, disp, h, beta, mu, hat, ld_out, conv, (int*)st, n_fallback, w), w ? "irls+wald" : "irls");
}

static int alpha_mle_op(pdq_ctx* c, const LaunchCfg& lc, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* mu,
                        int64_t ld_mu, const double* alpha_hat, double min_disp, double max_disp, double prior_disp_var,
                        const double* prior_var_dev, int cr_reg, int prior_reg, double* alpha, double* conv, int* status,
                        const double* hint_in = nullptr, double* hint_out = nullptr) {
    void* st = status;
    if (!st)
        if (int e = ensure(c, kBufStatus, (size_t)G * sizeof(int), &st)) return e;
    return done(c, launch_alpha_mle(lc, d, counts, ld, G, mu, ld_mu, alpha_hat, min_disp, max_disp, prior_disp_var, prior_var_dev, cr_reg,
                                    prior_reg, alpha, conv, (int*)st, hint_in, hint_out), "alpha_mle");
}

extern "C" int pdq_lin_reg_mu_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, double min_mu,
                                  double* mu_out, int64_t ld_out) {
    CHECK_CTX(c);
    if (!d || !counts || !mu_out || G <= 0 || ld < G || ld_out < G) return fail(c, PDQ_ERR_INVALID, "pdq_lin_reg_mu_dev: bad arguments");
    return done(c, launch_lin_reg_mu(cfg(c, G, d->d.N), d->d, counts, ld, G, min_mu, mu_out, ld_out), "lin_reg_mu");
}

extern "C" int pdq_irls_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, const double* disp,
                            double min_mu, double beta_tol, double min_beta, double max_beta, int maxiter, double* beta,
                            double* mu, double* hat, int64_t ld_out, double* conv, int* n_fallback_dev) {
    CHECK_CTX(c);
    if (!d || !counts || !disp || !beta || !mu || !hat || !conv || G <= 0 || ld < G || ld_out < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_irls_dev: bad arguments");
    return irls_op(c, cfg(c, G, d->d.N), d->d, counts, ld, G, disp, IrlsHost{min_mu, beta_tol, min_beta, max_beta, maxiter}, beta, mu, hat,
                   ld_out, conv, nullptr, n_fallback_dev);
}

extern "C" int pdq_irls_wald_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, const double* disp,
                                 double min_mu, double beta_tol, double min_beta, double max_beta, int maxiter, double* beta,
                                 double* mu, double* hat, int64_t ld_out, double* conv, int* n_fallback_dev, const double* ridge,
                                 const double* contrast, double lfc_null, int alt, double* pv, double* stat, double* se) {
    CHECK_CTX(c);
    if (!d || !counts || !disp || !beta || !mu || !hat || !conv || G <= 0 || ld < G || ld_out < G || !ridge || !contrast || !pv ||
        !stat || !se)
        return fail(c, PDQ_ERR_INVALID, "pdq_irls_wald_dev: bad arguments");
    if (int e = check_alt(c, alt, "pdq_irls_wald_dev: bad arguments")) return e;
    const WaldHost w{ridge, contrast, lfc_null, alt, pv, stat, se};
    return irls_op(c, cfg(c, G, d->d.N), d->d, counts, ld, G, disp, IrlsHost{min_mu, beta_tol, min_beta, max_beta, maxiter}, beta, mu, hat,
                   ld_out, conv, nullptr, n_fallback_dev, &w);
}

extern "C" int pdq_alpha_mle_hint_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, const double* mu,
                                      int64_t ld_mu, const double* alpha_hat, double min_disp, double max_disp, double prior_disp_var,
                                      const double* prior_var_dev, int cr_reg, int prior_reg, double* alpha, double* conv,
                                      const double* hint_in, double* hint_out) {
    CHECK_CTX(c);
    if (!d || !counts || !mu || !alpha_hat || !alpha || !conv || G <= 0 || ld < G || ld_mu < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_alpha_mle_dev: bad arguments");
    if (int e = check_prior(c, prior_reg, prior_var_dev, prior_disp_var)) return e;
    return alpha_mle_op(c, cfg(c, G, d->d.N), d->d, counts, ld, G, mu, ld_mu, alpha_hat, min_disp, max_disp, prior_disp_var, prior_var_dev,
                        cr_reg, prior_reg, alpha, conv, nullptr, hint_in, hint_out);
}

extern "C" int pdq_alpha_mle_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, const double* mu,
                                 int64_t ld_mu, const double* alpha_hat, double min_disp, double max_disp, double prior_disp_var,
                                 const double* prior_var_dev, int cr_reg, int prior_reg, double* alpha, double* conv) {
    return pdq_alpha_mle_hint_dev(c, d, counts, ld, G, mu, ld_mu, alpha_hat, min_disp, max_disp, prior_disp_var, prior_var_dev, cr_reg,
                                  prior_reg, alpha, conv, nullptr, nullptr);
}

extern "C" int pdq_map_irls_wald_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, const double* mu,
                                     int64_t ld_mu, const double* fitted, const double* genewise, const double* hint_in,
                                     const double* trend_out16, double min_disp, double max_disp, double prior_disp_var,
                                     const double* prior_var_dev, double* map, double* map_conv, double* disp, double* outlier,
                                     double min_mu, double beta_tol, double min_beta, double max_beta, int maxiter, double* beta,
                                     double* mu_out, double* hat, int64_t ld_out, double* conv, const double* ridge,
                                     const double* contrast, double lfc_null, int alt, double* pv, double* stat, double* se) {
    CHECK_CTX(c);
    if (!d || !counts || !mu || !fitted || !genewise || !hint_in || !trend_out16 || !map || !map_conv || !disp || !beta || !mu_out ||
        !hat || !conv || G <= 0 || ld < G || ld_mu < G || ld_out < G || !ridge || !contrast || !pv || !stat || !se)
        return fail(c, PDQ_ERR_INVALID, "pdq_map_irls_wald_dev: bad arguments");
    if (int e = check_alt(c, alt, "pdq_map_irls_wald_dev: bad arguments")) return e;
    if (!prior_var_dev && !(prior_disp_var > 0.0)) return fail(c, PDQ_ERR_INVALID, "pdq_map_irls_wald_dev: needs prior_disp_var > 0");
    // The hand-off pays where a warp works on few tiles per launch, so that the drained end of the search and the ramp-up of the
    // fit are a visible share of both: measured on H100 it gains 3-7 % up to ~10 tiles per resident warp of the search (12 per SM)
    // and loses 2.5 % at 20 (DESIGN.md §5).  Above 12 the three stages run as the three launches.
    const LaunchCfg lcfg = cfg(c, G, d->d.N);
    const IrlsHost h{min_mu, beta_tol, min_beta, max_beta, maxiter};
    const WaldHost w{ridge, contrast, lfc_null, alt, pv, stat, se};
    // wide designs (p > PDQ_MAX_P) have no fused pair: always the three launches
    if (many_tiles(lcfg, G) || d->d.p > PDQ_MAX_P) {
        if (int e = alpha_mle_op(c, lcfg, d->d, counts, ld, G, mu, ld_mu, fitted, min_disp, max_disp, prior_disp_var, prior_var_dev, 1, 1, map,
                                 map_conv, nullptr, hint_in, nullptr))
            return e;
        if (int e = done(c, launch_select_disp(lcfg, genewise, map, fitted, trend_out16, (size_t)G, min_disp, max_disp, disp, outlier),
                         "select_dispersions"))
            return e;
        return irls_op(c, lcfg, d->d, counts, ld, G, disp, h, beta, mu_out, hat, ld_out, conv, nullptr, nullptr, &w);
    }
    void* status;
    if (int e = ensure(c, kBufStatus, 2 * (size_t)G * sizeof(int), &status)) return e;
    if ((size_t)G > c->tile_cap) {  // one word per gene covers every tile size
        if (c->tile_done) {
            CU(c, cudaFree(c->tile_done));
            ++c->buf_epoch;
        }
        c->tile_done = nullptr;
        c->tile_cap = 0;
        const size_t want = (size_t)G + (size_t)G / 8 + 64;
        CU(c, cudaMalloc((void**)&c->tile_done, want * sizeof(unsigned)));
        CU(c, cudaMemsetAsync(c->tile_done, 0, want * sizeof(unsigned), c->stream));
        c->tile_cap = want;
    }
    if (!c->tail_err_host) {
        CU(c, cudaHostAlloc((void**)&c->tail_err_host, 8, cudaHostAllocMapped));
        *c->tail_err_host = 0;
        CU(c, cudaHostGetDevicePointer((void**)&c->tail_err_dev, c->tail_err_host, 0));
    }
    const TailHost t{mu, ld_mu, fitted, genewise, hint_in, trend_out16, min_disp, max_disp, prior_disp_var, prior_var_dev, map, map_conv,
                     disp, outlier, beta, mu_out, hat, conv, ld_out, (int*)status, (int*)status + G, c->tile_done, c->tail_err_dev};
    return done(c, launch_map_irls(lcfg, d->d, counts, ld, G, t, h, w), "map+irls+wald");
}

// 0 while every tile hand-off of pdq_map_irls_wald_dev completed; 1 + tile after a wait gave up (valid after a stream synchronisation)
extern "C" int pdq_map_irls_status(pdq_ctx* c, unsigned long long* status_out) {
    CHECK_CTX(c);
    if (!status_out) return fail(c, PDQ_ERR_INVALID, "pdq_map_irls_status: bad arguments");
    *status_out = c->tail_err_host ? *(volatile unsigned long long*)c->tail_err_host : 0ULL;
    return PDQ_OK;
}

extern "C" int pdq_wald_test_dev(pdq_ctx* c, const pdq_design* d, const double* disp, const double* lfc, const double* mu,
                                 int64_t ld_mu, int G, const double* ridge, const double* contrast, double lfc_null, int alt,
                                 double* pv, double* stat, double* se) {
    CHECK_CTX(c);
    if (!d || !disp || !lfc || !mu || !ridge || !contrast || !pv || !stat || !se || G <= 0 || ld_mu < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_wald_test_dev: bad arguments");
    if (int e = check_alt(c, alt, "pdq_wald_test_dev: bad arguments")) return e;
    return done(c, launch_wald(cfg(c, G, d->d.N), d->d, disp, lfc, mu, ld_mu, G, ridge, contrast, lfc_null, alt, pv, stat, se), "wald_test");
}

extern "C" int pdq_lfc_shrink_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, const double* size,
                                  double prior_no_shrink_scale, double prior_scale, int shrink_index, double* lfcs, double* inv_hessians,
                                  double* conv, int* status) {
    CHECK_CTX(c);
    if (!d || !counts || !size || !lfcs || !inv_hessians || !conv || !status || G <= 0 || ld < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_lfc_shrink_dev: bad arguments");
    if (int e = check_shrink(c, d->d.p, shrink_index, prior_no_shrink_scale, prior_scale)) return e;
    if (int e = design_width(c, d->d.p, true)) return e;  // also refuses a pack made before an opt-in was turned off
    return done(c, launch_lfc_shrink(cfg(c, G, d->d.N), d->d, counts, ld, G, size, prior_no_shrink_scale, prior_scale, shrink_index, lfcs,
                                     inv_hessians, conv, status), "lfc_shrink");
}

extern "C" int pdq_fp64_peak_tflops(pdq_ctx* c, double* tflops_out) {
    CHECK_CTX(c);
    if (!tflops_out) return fail(c, PDQ_ERR_INVALID, "pdq_fp64_peak_tflops: bad arguments");
    void* buf;
    if (int e = ensure(c, kBufA, (size_t)c->prop.multiProcessorCount * 8 * 256 * 8, &buf)) return e;
    const LaunchCfg lc = cfg(c, 1, 1);
    cudaEvent_t e0, e1;
    CU(c, cudaEventCreate(&e0));
    CU(c, cudaEventCreate(&e1));
    double flop = 0.0, best = 0.0;
    for (int rep = 0; rep < 4; ++rep) {  // first repetition warms up
        CU(c, cudaEventRecord(e0, c->stream));
        if (int e = done(c, launch_fp64_peak(lc, (double*)buf, 20000, &flop), "fp64_peak")) return e;
        CU(c, cudaEventRecord(e1, c->stream));
        CU(c, cudaEventSynchronize(e1));
        float ms = 0.f;
        CU(c, cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && ms > 0.f) best = fmax(best, flop / (ms * 1e-3) / 1e12);
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    *tflops_out = best;
    return PDQ_OK;
}

extern "C" int pdq_mom_dispersions_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, double min_disp,
                                       double max_disp, double* alpha, double* normed_mean, double min_mu, double* mu_hat_out,
                                       int64_t ld_mu) {
    CHECK_CTX(c);
    if (!d || !counts || !alpha || !normed_mean || G <= 0 || ld < G || (mu_hat_out && ld_mu < G))
        return fail(c, PDQ_ERR_INVALID, "pdq_mom_dispersions_dev: bad arguments");
    if (int e = check_not_square(c, d->d.N, d->d.p)) return e;
    return done(c, launch_mom_from_counts(cfg(c, G, d->d.N), d->d, counts, ld, G, min_disp, max_disp, alpha, normed_mean, min_mu, mu_hat_out, ld_mu),
                "mom_dispersions");
}

extern "C" int pdq_mom_alpha_mle_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, double min_disp,
                                     double max_disp, double min_mu, double* mom, double* normed_mean, double* mu_hat, int64_t ld_mu,
                                     double* alpha, double* conv, double* hint_out) {
    CHECK_CTX(c);
    if (!d || !counts || !mom || !normed_mean || !mu_hat || !alpha || !conv || G <= 0 || ld < G || ld_mu < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_mom_alpha_mle_dev: bad arguments");
    if (int e = check_not_square(c, d->d.N, d->d.p)) return e;
    void* status;
    if (int e = ensure(c, kBufStatus, (size_t)G * sizeof(int), &status)) return e;
    // The fold pays where a warp works on few tiles per launch, as the MAP -> LFC hand-off does: the start values then run at the
    // search's occupancy (3 blocks per SM) instead of their own, which costs more than the saved drain and ramp-up once the
    // streaming is long.  Whole resident pass on H100: 3 % faster at C2 (3.2 tiles per resident search warp), 6 % slower at the C5
    // shard (19.7) (DESIGN.md §5).  Above 12 tiles the two launches, as in pdq_map_irls_wald_dev.
    const LaunchCfg lcfg = cfg(c, G, d->d.N);
    if (many_tiles(lcfg, G)) {
        if (int e = done(c, launch_mom_from_counts(lcfg, d->d, counts, ld, G, min_disp, max_disp, mom, normed_mean, min_mu, mu_hat, ld_mu),
                         "mom_dispersions"))
            return e;
        return alpha_mle_op(c, lcfg, d->d, counts, ld, G, mu_hat, ld_mu, mom, min_disp, max_disp, 1.0, nullptr, 1, 0, alpha, conv, (int*)status,
                            nullptr, hint_out);
    }
    return done(c, launch_mom_alpha(lcfg, d->d, counts, ld, G, min_disp, max_disp, min_mu, mom, normed_mean, mu_hat, ld_mu,
                                    alpha, conv, (int*)status, hint_out),
                "mom_alpha_mle");
}

extern "C" int pdq_mu_from_lfc_dev(pdq_ctx* c, const pdq_design* d, const double* lfc, int G, double* mu, int64_t ld_out) {
    CHECK_CTX(c);
    if (!d || !lfc || !mu || G <= 0 || ld_out < G) return fail(c, PDQ_ERR_INVALID, "pdq_mu_from_lfc_dev: bad arguments");
    return done(c, launch_mu_from_lfc(cfg(c, G, d->d.N), d->d, lfc, G, mu, ld_out), "mu_from_lfc");
}

extern "C" int pdq_trend_fit_dev(pdq_ctx* c, const double* means, const double* genewise, size_t n, double min_disp, double max_disp,
                                 double trigamma_c, double* out16, double* fitted) {
    CHECK_CTX(c);
    if (!means || !genewise || !out16 || n == 0) return fail(c, PDQ_ERR_INVALID, "pdq_trend_fit_dev: bad arguments");
    void* scratch;
    if (int e = ensure(c, kBufRes, 3 * n * 8, &scratch)) return e;
    LaunchCfg lc{c->stream, 0, c->prop.multiProcessorCount, c->tickets, c->debug, c->grid_scratch};
    if (int e = done(c, launch_trend_fit(lc, means, genewise, (double*)scratch, n, 1, min_disp, max_disp, 1, min_disp, trigamma_c, 1, out16),
                     "trend_fit"))
        return e;
    if (fitted) return done(c, launch_trend_eval(lc, means, n, out16, fitted), "trend_eval");
    return PDQ_OK;
}

extern "C" int pdq_cooks_dev(pdq_ctx* c, const pdq_design* d, const int64_t* counts, int64_t ld, int G, const double* mu, const double* hat,
                             int64_t ld2, double cutoff, double* cooks_out, int64_t ld_out, double* robust_disp_out, double* outlier_out,
                             double* replaced_out) {
    CHECK_CTX(c);
    if (!d || !counts || !mu || !hat || !robust_disp_out || !outlier_out || !replaced_out || G <= 0 || ld < G || ld2 < G ||
        (cooks_out && ld_out < G))
        return fail(c, PDQ_ERR_INVALID, "pdq_cooks_dev: bad arguments");
    void* ws = nullptr;
    if (const size_t bytes = cooks_ws_bytes(d->d, G))
        if (int e = ensure(c, kBufCooks, bytes, &ws)) return e;
    return done(c, launch_cooks(cfg(c, G, d->d.N), d->d, counts, ld, G, mu, hat, ld2, cutoff, cooks_out, ld_out, robust_disp_out, outlier_out,
                                replaced_out, (double*)ws), "cooks");
}

extern "C" int pdq_size_factors_dev(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, double* sf_out, double* logmeans_out) {
    CHECK_CTX(c);
    if (!counts || !sf_out || N <= 0 || G <= 0 || ld < G) return fail(c, PDQ_ERR_INVALID, "pdq_size_factors_dev: bad arguments");
    void *lm = logmeans_out, *scratch;
    if (!lm)
        if (int e = ensure(c, kBufF, (size_t)G * 8, &lm)) return e;
    if (int e = ensure(c, kBufB, (size_t)N * G * 8, &scratch)) return e;
    return done(c, launch_size_factors_ex(cfg(c, G, N), counts, ld, N, G, 0 /* ratio */, nullptr, (double*)lm, nullptr, (double*)scratch, sf_out),
                "size_factors");
}

static int sf_ex_check(pdq_ctx* c, const void* counts, const void* sf_out, int64_t ld, int N, int G, int kind, const char* what) {
    if (!counts || !sf_out || N <= 0 || G <= 0 || ld < G) return fail(c, PDQ_ERR_INVALID, "%s: bad arguments", what);
    if (kind != 0 && kind != 1) return fail(c, PDQ_ERR_INVALID, "%s: unknown kind %d (0 ratio, 1 poscounts)", what, kind);
    return PDQ_OK;
}

extern "C" int pdq_size_factors_ex_dev(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, int kind, const uint8_t* control,
                                       double* sf_out, double* logmeans_out) {
    CHECK_CTX(c);
    if (int e = sf_ex_check(c, counts, sf_out, ld, N, G, kind, "pdq_size_factors_ex_dev")) return e;
    void *lm = logmeans_out, *kept, *scratch;
    if (!lm)
        if (int e = ensure(c, kBufF, (size_t)G * 8, &lm)) return e;
    if (int e = ensure(c, kBufC, (size_t)G * 8, &kept)) return e;
    if (int e = ensure(c, kBufB, (size_t)N * G * 8, &scratch)) return e;
    return done(c, launch_size_factors_ex(cfg(c, G, N), counts, ld, N, G, kind, control, (double*)lm, (double*)kept, (double*)scratch,
                                          sf_out),
                "size_factors_ex");
}

extern "C" int pdq_size_factors_from_logmeans_dev(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, const double* logmeans,
                                                  double* sf_out) {
    CHECK_CTX(c);
    if (!counts || !logmeans || !sf_out || N <= 0 || G <= 0 || ld < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_size_factors_from_logmeans_dev: bad arguments");
    void* scratch;
    if (int e = ensure(c, kBufB, (size_t)N * G * 8, &scratch)) return e;
    return done(c, launch_size_factors_from_logmeans(cfg(c, G, N), counts, ld, N, G, logmeans, (double*)scratch, sf_out),
                "size_factors_from_logmeans");
}

static int vst_check(pdq_ctx* c, const void* counts, const void* sf, const void* out, int64_t ld, int N, int G, int kind, double c0,
                     int64_t ld_out, const char* what) {
    if (!counts || !sf || !out || N <= 0 || G <= 0 || ld < G || ld_out < G) return fail(c, PDQ_ERR_INVALID, "%s: bad arguments", what);
    if (kind != 0 && kind != 1) return fail(c, PDQ_ERR_INVALID, "%s: unknown kind %d (0 parametric, 1 mean)", what, kind);
    if (!(c0 > 0.0)) return fail(c, PDQ_ERR_INVALID, "%s: %s must be > 0", what, kind == 0 ? "a0" : "the mean dispersion");
    return PDQ_OK;
}

extern "C" int pdq_vst_transform_dev(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, const double* size_factors, int kind,
                                     double c0, double c1, double* out, int64_t ld_out) {
    CHECK_CTX(c);
    if (int e = vst_check(c, counts, size_factors, out, ld, N, G, kind, c0, ld_out, "pdq_vst_transform_dev")) return e;
    return done(c, launch_vst_transform(cfg(c, G, N), counts, ld, N, G, size_factors, kind, c0, c1, out, ld_out), "vst_transform");
}

extern "C" int pdq_gather_columns_dev(pdq_ctx* c, const double* in, int64_t ld_in, int N, const int* idx_dev, int R, double* out,
                                      int64_t ld_out) {
    CHECK_CTX(c);
    if (!in || !idx_dev || !out || N <= 0 || R < 0 || ld_out < R) return fail(c, PDQ_ERR_INVALID, "pdq_gather_columns_dev: bad arguments");
    const int rc = launch_gather_cols(c->stream, in, ld_in, N, idx_dev, R, out, ld_out);
    return done(c, rc, "gather_columns");
}

extern "C" int pdq_column_sums_dev(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, double* sums_out) {
    CHECK_CTX(c);
    if (!counts || !sums_out || N <= 0 || G <= 0 || ld < G) return fail(c, PDQ_ERR_INVALID, "pdq_column_sums_dev: bad arguments");
    return done(c, launch_column_sums(c->stream, counts, ld, N, G, sums_out), "column_sums");
}

extern "C" int pdq_scatter_rows_dev(pdq_ctx* c, const double* in, double* out, const int* perm_dev, int n, int nvec, int64_t stride, int width) {
    CHECK_CTX(c);
    if (!in || !out || !perm_dev || n < 0 || nvec < 1 || width < 1 || stride < n) return fail(c, PDQ_ERR_INVALID, "pdq_scatter_rows_dev: bad arguments");
    return done(c, launch_scatter_rows(c->stream, in, out, perm_dev, n, nvec, stride, width), "scatter_rows");
}

extern "C" int pdq_scatter_segments_dev(pdq_ctx* c, const double* in, double* out, const int* src_dev, int nseg, const int64_t* seg) {
    CHECK_CTX(c);
    if (!in || !out || !seg || nseg < 1 || nseg > kMaxScatterSegs) return fail(c, PDQ_ERR_INVALID, "pdq_scatter_segments_dev: bad arguments");
    for (int i = 0; i < nseg; ++i)
        if (seg[4 * i] < 0 || seg[4 * i + 1] < 0 || seg[4 * i + 1] > INT32_MAX || seg[4 * i + 2] < 1 || seg[4 * i + 2] > INT32_MAX ||
            (seg[4 * i + 3] && !src_dev))
            return fail(c, PDQ_ERR_INVALID, "pdq_scatter_segments_dev: bad segment %d", i);
    // page-locked host memory is written through its device address (the same pointer under unified addressing)
    cudaPointerAttributes at{};
    CU(c, cudaPointerGetAttributes(&at, out));
    if (at.type == cudaMemoryTypeHost) {
        if (!at.devicePointer) return fail(c, PDQ_ERR_INVALID, "pdq_scatter_segments_dev: host `out` is not mapped into the device");
        out = static_cast<double*>(at.devicePointer);
    } else if (at.type == cudaMemoryTypeUnregistered) {
        return fail(c, PDQ_ERR_INVALID, "pdq_scatter_segments_dev: `out` is pageable host memory");
    }
    return done(c, launch_scatter_segments(c->stream, in, out, src_dev, nseg, seg), "scatter_segments");
}

extern "C" int pdq_select_dispersions_dev(pdq_ctx* c, const double* genewise, const double* map, const double* fitted,
                                          const double* trend_out16, size_t n, double min_disp, double max_disp, double* disp_out,
                                          double* outlier_out) {
    CHECK_CTX(c);
    if (!genewise || !map || !fitted || !trend_out16 || !disp_out || n == 0)
        return fail(c, PDQ_ERR_INVALID, "pdq_select_dispersions_dev: bad arguments");
    LaunchCfg lc{c->stream, 0, c->prop.multiProcessorCount, c->tickets, c->debug, c->grid_scratch};
    return done(c, launch_select_disp(lc, genewise, map, fitted, trend_out16, n, min_disp, max_disp, disp_out, outlier_out), "select_dispersions");
}

// --------------------------------------------------------------------------------------------- host-buffer ops
// ---- host <-> device copies of caller buffers ------------------------------------------------------------------
// numpy arrays are pageable; a plain cudaMemcpy from/to pageable memory is staged by the driver at a fraction of the
// PCIe rate.  Large pageable buffers are therefore pipelined through two page-locked chunks owned by the context:
// a few host threads copy chunk k+1 into / out of the ring while the DMA engine moves chunk k.
static const size_t kStageChunk = 8u << 20;

static bool is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

static void par_memcpy(void* dst, const void* src, size_t n) {
    const int nt = n >= (2u << 20) ? 8 : 1;
    HostPool::get().run(nt, [&](int t, int k) {
        const size_t lo = n * t / k, hi = n * (t + 1) / k;
        memcpy((char*)dst + lo, (const char*)src + lo, hi - lo);
    });
}

static int stage_init(pdq_ctx* c) {
    for (int i = 0; i < 2; ++i)
        if (!c->stage[i]) {
            CU(c, cudaHostAlloc(&c->stage[i], kStageChunk, cudaHostAllocDefault));
            CU(c, cudaEventCreateWithFlags(&c->stage_ev[i], cudaEventDisableTiming));
        }
    return 0;
}

static int copy_h2d(pdq_ctx* c, void* dst, const void* src, size_t bytes) {
    if (!c->staging || bytes < (1u << 20) || is_pinned(src)) {
        CU(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->stream));
        return 0;
    }
    if (int e = stage_init(c)) return e;
    int k = 0;
    for (size_t off = 0; off < bytes; off += kStageChunk, k ^= 1) {
        const size_t n = bytes - off < kStageChunk ? bytes - off : kStageChunk;
        if (c->stage_busy[k]) CU(c, cudaEventSynchronize(c->stage_ev[k]));
        par_memcpy(c->stage[k], (const char*)src + off, n);
        CU(c, cudaMemcpyAsync((char*)dst + off, c->stage[k], n, cudaMemcpyHostToDevice, c->stream));
        CU(c, cudaEventRecord(c->stage_ev[k], c->stream));
        c->stage_busy[k] = true;
    }
    return 0;
}

// device -> caller buffer; the pageable path synchronises the stream chunk by chunk
static int copy_d2h(pdq_ctx* c, void* dst, const void* src, size_t bytes) {
    if (!c->staging || bytes < (1u << 20) || is_pinned(dst)) {
        CU(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
        return 0;
    }
    if (int e = stage_init(c)) return e;
    for (int i = 0; i < 2; ++i)
        if (c->stage_busy[i]) {
            CU(c, cudaEventSynchronize(c->stage_ev[i]));
            c->stage_busy[i] = false;
        }
    const size_t nchunks = (bytes + kStageChunk - 1) / kStageChunk;
    for (size_t i = 0; i <= nchunks; ++i) {
        if (i < nchunks) {  // launch DMA of chunk i into slot i&1
            const size_t off = i * kStageChunk, n = bytes - off < kStageChunk ? bytes - off : kStageChunk;
            CU(c, cudaMemcpyAsync(c->stage[i & 1], (const char*)src + off, n, cudaMemcpyDeviceToHost, c->stream));
            CU(c, cudaEventRecord(c->stage_ev[i & 1], c->stream));
        }
        if (i > 0) {  // drain chunk i-1 while chunk i is in flight
            const size_t j = i - 1, off = j * kStageChunk, n = bytes - off < kStageChunk ? bytes - off : kStageChunk;
            CU(c, cudaEventSynchronize(c->stage_ev[j & 1]));
            par_memcpy((char*)dst + off, c->stage[j & 1], n);
        }
    }
    return 0;
}

static int h2d_2d(pdq_ctx* c, void* dst, const void* src, int64_t ld, int N, int G, size_t elem) {
    if (ld == G) return copy_h2d(c, dst, src, (size_t)N * G * elem);
    CU(c, cudaMemcpy2DAsync(dst, (size_t)G * elem, src, (size_t)ld * elem, (size_t)G * elem, N, cudaMemcpyHostToDevice, c->stream));
    return 0;
}

// ---- residency: content-addressed device copies of the (N, G) buffers ------------------------------------------------
// One deseq2() hands the backend the SAME counts four times (dds.py:752 / 759, 779, 902, 954), the same mu_hat twice and the
// mu it got back from the LFC fit once more (ds.py:338) -- each time as a fresh host array, so pointer identity says nothing.
// The entry points therefore key device copies on a 128-bit checksum of the FULL content, computed at memory bandwidth by a
// few host threads; an (N, G) OUTPUT is kept on the device under the same checksum, computed there by a reduction kernel, so
// that handing it back costs a checksum instead of an upload.  A hit replaces a PCIe transfer (slower still from pageable memory)
// by a read of host memory.  Never by pointer, never by a sample of the content.  PDQ_RESIDENCY=0 switches it off.
static const size_t kResMinBytes = 1u << 20;
static const int kHashSlots = 8;

static inline uint64_t hash_a(uint64_t w, uint64_t i) {
    uint64_t t = (w + (i + 1) * 0x9E3779B97F4A7C15ull) * 0xBF58476D1CE4E5B9ull;
    return t ^ (t >> 31);
}
static inline uint64_t hash_b(uint64_t w, uint64_t i) {
    uint64_t u = (w ^ ((i + 1) * 0xD6E8FEB86659FD93ull)) * 0x94D049BB133111EBull;
    return u ^ (u >> 29);
}

// sum over the 64-bit words of the buffer of two position-dependent mixes (wrapping): order-free, so host threads and device
// blocks may reduce in any order and agree bit for bit
static void host_hash(const void* p, size_t bytes, uint64_t out[2]) {
    const uint64_t* w = (const uint64_t*)p;
    const size_t n = bytes / 8;
    int nt = (int)(bytes >> 20);  // one thread per MB, up to the pool: enough to reach the memory bandwidth of a socket
    if (nt < 1) nt = 1;
    uint64_t part[64][2] = {};
    HostPool::get().run(nt > 32 ? 32 : nt, [&](int t, int k) {
        const size_t lo = n * t / k, hi = n * (t + 1) / k;
        uint64_t a = 0, b = 0;
        for (size_t i = lo; i < hi; ++i) {
            a += hash_a(w[i], (uint64_t)i);
            b += hash_b(w[i], (uint64_t)i);
        }
        part[t][0] = a;
        part[t][1] = b;
    });
    out[0] = out[1] = 0;
    for (int t = 0; t < 64; ++t) {
        out[0] += part[t][0];
        out[1] += part[t][1];
    }
}

// entry states: 0 = spare allocation, 1 = being filled by the running call (becomes valid when that call succeeds), 2 = valid
typedef pdq_ctx::ResEntry ResEntry;

static void res_begin(pdq_ctx* c) {
    ++c->res_call;
    for (auto* e : c->res)
        if (e->state == 1) e->state = 0;  // left behind by a call that failed: never addressable
}

// a cache-owned buffer of `bytes` in state "filling": a spare of that size, else a new allocation (evicting least recently used
// entries of other calls while the byte budget or the entry limit is exceeded); nullptr when nothing fits
static ResEntry* res_new_entry(pdq_ctx* c, size_t bytes) {
    if (bytes > c->res_cap / 2) return nullptr;
    ResEntry* k = nullptr;
    for (auto* e : c->res)
        if (e->state == 0 && e->bytes == bytes) k = e;
    while (!k && (c->res_bytes + bytes > c->res_cap || c->res.size() >= 16)) {
        int lru = -1;
        for (size_t i = 0; i < c->res.size(); ++i) {
            const ResEntry* e = c->res[i];
            if (e->call == c->res_call && e->state != 0) continue;  // in use by the running call
            if (lru < 0 || (e->state == 0 && c->res[lru]->state != 0) ||
                ((e->state == 0) == (c->res[lru]->state == 0) && e->stamp < c->res[lru]->stamp))
                lru = (int)i;
        }
        if (lru < 0) return nullptr;
        ResEntry* v = c->res[lru];
        if (v->bytes == bytes) {  // same size: take the allocation over instead of free + malloc
            k = v;
            break;
        }
        if (cudaFree(v->dptr) != cudaSuccess) return nullptr;
        c->res_bytes -= v->bytes;
        c->res.erase(c->res.begin() + lru);
        delete v;
    }
    if (!k) {
        void* p = nullptr;
        if (cudaMalloc(&p, bytes) != cudaSuccess) {
            cudaGetLastError();
            return nullptr;
        }
        k = new ResEntry();
        k->dptr = p;
        k->bytes = bytes;
        c->res.push_back(k);
        c->res_bytes += bytes;
    }
    k->h[0] = k->h[1] = 0;
    k->pending = -1;
    k->state = 1;
    k->call = c->res_call;
    k->stamp = ++c->res_clock;
    return k;
}

static bool res_on(const pdq_ctx* c, int64_t ld, int G, size_t bytes) { return c->residency && ld == G && bytes >= kResMinBytes && bytes % 8 == 0; }

// Device buffer holding the caller's (N, G) input.  *need_upload = the caller still has to fill it (cache miss, or cache off:
// then `scratch` names the context buffer used instead).
static int res_input(pdq_ctx* c, const void* host, int64_t ld, int N, int G, size_t elem, int scratch, void** dptr, bool* need_upload) {
    const size_t bytes = (size_t)N * G * elem;
    *need_upload = true;
    if (res_on(c, ld, G, bytes)) {
        uint64_t h[2];
        host_hash(host, bytes, h);
        for (auto* e : c->res)
            if (e->state == 2 && e->bytes == bytes && e->h[0] == h[0] && e->h[1] == h[1]) {
                e->stamp = ++c->res_clock;
                e->call = c->res_call;
                *dptr = e->dptr;
                *need_upload = false;
                ++c->res_hits;
                c->res_hit_bytes += (int64_t)bytes;
                return 0;
            }
        if (ResEntry* k = res_new_entry(c, bytes)) {
            k->h[0] = h[0];
            k->h[1] = h[1];
            *dptr = k->dptr;
            ++c->res_misses;
            return 0;
        }
    }
    return ensure(c, scratch, bytes, dptr);
}

// Device buffer for an (N, G) OUTPUT; *slot != nullptr when it is cache-owned (then call res_commit once the kernels are enqueued)
static int res_output(pdq_ctx* c, size_t bytes, int scratch, void** dptr, ResEntry** slot) {
    *slot = nullptr;
    if (c->residency && bytes >= kResMinBytes && bytes % 8 == 0 && c->hash_pending < kHashSlots) {
        if (ResEntry* k = res_new_entry(c, bytes)) {
            *dptr = k->dptr;
            *slot = k;
            return 0;
        }
    }
    return ensure(c, scratch, bytes, dptr);
}

// checksum of a finished output on the device (same function as host_hash), delivered to the host with the call's final sync
static int res_commit(pdq_ctx* c, ResEntry* e) {
    if (!e) return 0;
    if (!c->hash_dev) {
        CU(c, cudaMalloc((void**)&c->hash_dev, 2 * kHashSlots * 8));
        CU(c, cudaHostAlloc((void**)&c->hash_host, 2 * kHashSlots * 8, cudaHostAllocDefault));
    }
    const int q = c->hash_pending++;
    e->pending = q;
    CU(c, cudaMemsetAsync(c->hash_dev + 2 * q, 0, 16, c->stream));
    if (launch_hash(c->stream, c->prop.multiProcessorCount, e->dptr, e->bytes / 8, c->hash_dev + 2 * q) < 0)
        return fail(c, PDQ_ERR_CUDA, "hash kernel launch failed");
    ++c->launches;
    CU(c, cudaMemcpyAsync(c->hash_host + 2 * q, c->hash_dev + 2 * q, 16, cudaMemcpyDeviceToHost, c->stream));
    return 0;
}

// the call succeeded and its stream is synchronised: inputs uploaded and outputs written by it become addressable
static void res_finalize(pdq_ctx* c) {
    for (auto* e : c->res) {
        if (e->state != 1 || e->call != c->res_call) continue;
        if (e->pending >= 0) {
            e->h[0] = c->hash_host[2 * e->pending];
            e->h[1] = c->hash_host[2 * e->pending + 1];
            e->pending = -1;
        }
        e->state = 2;
        for (auto* o : c->res)  // the same content from an earlier call: keep one copy, the other becomes a spare
            if (o != e && o->state == 2 && o->bytes == e->bytes && o->h[0] == e->h[0] && o->h[1] == e->h[1]) o->state = 0;
    }
    c->hash_pending = 0;
}

extern "C" int pdq_residency_stats(const pdq_ctx* c, int64_t* hits, int64_t* misses, int64_t* hit_bytes, int64_t* resident_bytes) {
    if (!c) return PDQ_ERR_INVALID;
    if (hits) *hits = c->res_hits;
    if (misses) *misses = c->res_misses;
    if (hit_bytes) *hit_bytes = c->res_hit_bytes;
    if (resident_bytes) *resident_bytes = (int64_t)c->res_bytes;
    return PDQ_OK;
}

extern "C" int pdq_residency_clear(pdq_ctx* c) {
    CHECK_CTX(c);
    CU(c, cudaStreamSynchronize(c->stream));
    for (auto* e : c->res) {
        if (e->dptr) cudaFree(e->dptr);
        delete e;
    }
    c->res.clear();
    c->res_bytes = 0;
    c->hash_pending = 0;
    return PDQ_OK;
}

// ---- gene-block pipeline --------------------------------------------------------------------------------------
// The plugin calls move 32-64 MB each way around a sub-millisecond kernel.  When every large host buffer is page-locked the call
// is split into gene blocks on two streams: the column block k+1 is uploaded while block k computes and block k-1 is
// downloaded (PCIe is full duplex, the kernels take `ld`, so a block is just a pointer offset).  Per-gene results do not
// depend on the split (different lane-group widths only change the order of the floating-point sums).
static const int kPipeMaxBlocks = 16;  // PDQ_PIPELINE=<blocks> (0/1 = off)

struct Pipe {
    pdq_ctx* c;
    bool on;
    int nb, G, Gb;
    int g0(int b) const { return b * Gb; }
    int gb(int b) const { return (b == nb - 1) ? G - b * Gb : Gb; }
    cudaStream_t st(int b) const { return on ? c->pstream[b & 1] : c->stream; }
    LaunchCfg cfg_for(int b, int N) const {
        // lane-group width from the WHOLE call's gene count, not the block's: per-gene results then do not depend on whether (and
        // how) a call was split -- only the width of the lane group fixes the order of a gene's floating-point sums
        LaunchCfg lc = cfg(c, G, N);
        lc.stream = st(b);
        lc.tickets = c->tickets + (on ? 4 * (1 + (b & 1)) : 0);
        return lc;
    }
};

static int pipe_begin(pdq_ctx* c, int G, std::initializer_list<const void*> big_host, Pipe* p) {
    const int want = c->pipeline > kPipeMaxBlocks ? kPipeMaxBlocks : c->pipeline;
    bool on = want > 1 && c->staging && G >= 4096;
    for (const void* h : big_host) on = on && (h == nullptr || is_pinned(h));  // nullptr: not transferred (resident already)
    p->c = c;
    p->on = on;
    p->G = G;
    p->nb = on ? want : 1;
    p->Gb = on ? (((G + want - 1) / want + 15) & ~15) : G;
    if (on) {
        while (p->nb > 1 && (p->nb - 1) * p->Gb >= G) --p->nb;
        CU(c, cudaEventRecord(c->pfork, c->stream));
        CU(c, cudaStreamWaitEvent(c->pstream[0], c->pfork, 0));
        CU(c, cudaStreamWaitEvent(c->pstream[1], c->pfork, 0));
    }
    return 0;
}

// joins the block streams back into c->stream (small per-gene vectors are moved whole on c->stream, before the fork and
// after the join: they may be pageable, and a pageable async copy blocks the host until the stream reaches it)
static int pipe_join(pdq_ctx* c, const Pipe& p) {
    if (p.on) {
        for (int i = 0; i < 2; ++i) {
            CU(c, cudaEventRecord(c->pjoin[i], c->pstream[i]));
            CU(c, cudaStreamWaitEvent(c->stream, c->pjoin[i], 0));
        }
    }
    return 0;
}

// end of a host-buffer call: join the block streams, checksum the cache-owned outputs, synchronise, publish the cache entries
static int call_end(pdq_ctx* c, const Pipe* p, std::initializer_list<pdq_ctx::ResEntry*> out_slots) {
    if (p)
        if (int e = pipe_join(c, *p)) return e;
    for (pdq_ctx::ResEntry* s : out_slots)
        if (int e = res_commit(c, s)) return e;
    CU(c, cudaStreamSynchronize(c->stream));
    res_finalize(c);
    return PDQ_OK;
}

// column block [g0, g0+gb) of an (N, G) array, host pitch ld_h elements <-> device pitch ld_d elements
static int cols_h2d(pdq_ctx* c, const Pipe& p, int b, void* dev, int64_t ld_d, const void* host, int64_t ld_h, int N, size_t elem) {
    if (!p.on) return h2d_2d(c, dev, host, ld_h, N, p.G, elem);
    CU(c, cudaMemcpy2DAsync((char*)dev + (size_t)p.g0(b) * elem, (size_t)ld_d * elem, (const char*)host + (size_t)p.g0(b) * elem,
                            (size_t)ld_h * elem, (size_t)p.gb(b) * elem, N, cudaMemcpyHostToDevice, p.st(b)));
    return 0;
}
static int cols_d2h(pdq_ctx* c, const Pipe& p, int b, void* host, int64_t ld_h, const void* dev, int64_t ld_d, int N, size_t elem) {
    if (!p.on && ld_h == p.G && ld_d == p.G) return copy_d2h(c, host, dev, (size_t)N * p.G * elem);
    CU(c, cudaMemcpy2DAsync((char*)host + (size_t)p.g0(b) * elem, (size_t)ld_h * elem, (const char*)dev + (size_t)p.g0(b) * elem,
                            (size_t)ld_d * elem, (size_t)p.gb(b) * elem, N, cudaMemcpyDeviceToHost, p.st(b)));
    return 0;
}
static int vec_h2d(pdq_ctx* c, void* dev, const void* host, size_t bytes) {
    CU(c, cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, c->stream));
    return 0;
}
static int vec_d2h(pdq_ctx* c, void* host, const void* dev, size_t bytes) {
    CU(c, cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, c->stream));
    return 0;
}

extern "C" int pdq_lin_reg_mu(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, const double* sf, const double* X, int p,
                              double min_mu, double* mu_out) {
    CHECK_CTX(c);
    if (!counts || !sf || !X || !mu_out || N <= 0 || G <= 0 || ld < G) return fail(c, PDQ_ERR_INVALID, "pdq_lin_reg_mu: bad arguments");
    pdq_design* d;
    if (int e = cached_design(c, X, sf, N, p, &d)) return e;
    void *dc, *dm;
    const size_t ng = (size_t)N * G;
    res_begin(c);
    bool up_c;
    pdq_ctx::ResEntry* slot_m;
    if (int e = res_input(c, counts, ld, N, G, 8, kBufCounts, &dc, &up_c)) return e;
    if (int e = res_output(c, ng * 8, kBufA, &dm, &slot_m)) return e;
    Pipe pp;
    if (int e = pipe_begin(c, G, {up_c ? (const void*)counts : nullptr, mu_out}, &pp)) return e;
    for (int b = 0; b < pp.nb; ++b) {
        if (up_c)
            if (int e = cols_h2d(c, pp, b, dc, G, counts, ld, N, 8)) return e;
        if (int e = done(c, launch_lin_reg_mu(pp.cfg_for(b, N), d->d, (const int64_t*)dc + pp.g0(b), G, pp.gb(b), min_mu,
                                              (double*)dm + pp.g0(b), G), "lin_reg_mu"))
            return e;
        if (int e = cols_d2h(c, pp, b, mu_out, G, dm, G, N, 8)) return e;
    }
    return call_end(c, &pp, {slot_m});
}

extern "C" int pdq_irls(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, const double* sf, const double* X, int p,
                        const double* disp, double min_mu, double beta_tol, double min_beta, double max_beta, int maxiter,
                        double* beta_out, double* mu_out, double* hat_out, double* conv_out, int* n_fallback) {
    CHECK_CTX(c);
    if (!counts || !sf || !X || !disp || !beta_out || !mu_out || !hat_out || !conv_out || N <= 0 || G <= 0 || ld < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_irls: bad arguments");
    pdq_design* d;
    if (int e = cached_design(c, X, sf, N, p, &d)) return e;
    const size_t ng = (size_t)N * G;
    void *dc, *dmu, *dhat, *ddisp, *dbeta, *dconv, *dmisc;
    res_begin(c);
    bool up_c;
    pdq_ctx::ResEntry *slot_mu, *slot_hat;
    if (int e = res_input(c, counts, ld, N, G, 8, kBufCounts, &dc, &up_c)) return e;
    if (int e = res_output(c, ng * 8, kBufA, &dmu, &slot_mu)) return e;
    if (int e = res_output(c, ng * 8, kBufB, &dhat, &slot_hat)) return e;
    if (int e = ensure(c, kBufC, (size_t)G * 8, &ddisp)) return e;
    if (int e = ensure(c, kBufD, (size_t)G * p * 8, &dbeta)) return e;
    if (int e = ensure(c, kBufE, (size_t)G * 8, &dconv)) return e;
    if (int e = ensure(c, kBufMisc, 64, &dmisc)) return e;
    void* status;
    if (int e = ensure(c, kBufStatus, (size_t)G * sizeof(int), &status)) return e;
    const IrlsHost h{min_mu, beta_tol, min_beta, max_beta, maxiter};
    Pipe pp;
    if (int e = vec_h2d(c, ddisp, disp, (size_t)G * 8)) return e;
    if (int e = pipe_begin(c, G, {up_c ? (const void*)counts : nullptr, mu_out, hat_out}, &pp)) return e;
    int nfb[kPipeMaxBlocks] = {};
    for (int b = 0; b < pp.nb; ++b) {
        const int g0 = pp.g0(b), gb = pp.gb(b);
        if (up_c)
            if (int e = cols_h2d(c, pp, b, dc, G, counts, ld, N, 8)) return e;
        if (int e = irls_op(c, pp.cfg_for(b, N), d->d, (const int64_t*)dc + g0, G, gb, (const double*)ddisp + g0, h,
                            (double*)dbeta + (size_t)g0 * p, (double*)dmu + g0, (double*)dhat + g0, G, (double*)dconv + g0,
                            (int*)status + g0, (int*)dmisc + b))
            return e;
        if (int e = cols_d2h(c, pp, b, mu_out, G, dmu, G, N, 8)) return e;
        if (int e = cols_d2h(c, pp, b, hat_out, G, dhat, G, N, 8)) return e;
    }
    if (int e = pipe_join(c, pp)) return e;
    if (int e = vec_d2h(c, beta_out, dbeta, (size_t)G * p * 8)) return e;
    if (int e = vec_d2h(c, conv_out, dconv, (size_t)G * 8)) return e;
    if (int e = vec_d2h(c, nfb, dmisc, (size_t)pp.nb * sizeof(int))) return e;
    if (int e = call_end(c, nullptr, {slot_mu, slot_hat})) return e;
    if (n_fallback) {
        *n_fallback = 0;
        for (int b = 0; b < pp.nb; ++b) *n_fallback += nfb[b];
    }
    return PDQ_OK;
}

extern "C" int pdq_alpha_mle(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, const double* X, int p, const double* mu,
                             int64_t ld_mu, const double* alpha_hat, double min_disp, double max_disp, double prior_disp_var,
                             int cr_reg, int prior_reg, double* alpha_out, double* conv_out) {
    CHECK_CTX(c);
    if (!counts || !X || !mu || !alpha_hat || !alpha_out || !conv_out || N <= 0 || G <= 0 || ld < G || ld_mu < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_alpha_mle: bad arguments");
    if (int e = design_width(c, p)) return e;
    if (int e = check_prior(c, prior_reg, nullptr, prior_disp_var)) return e;
    pdq_design* d;
    if (int e = cached_design(c, X, nullptr, N, p, &d)) return e;
    void *dc, *dmu, *dah, *dal, *dconv;
    res_begin(c);
    bool up_c, up_m;
    if (int e = res_input(c, counts, ld, N, G, 8, kBufCounts, &dc, &up_c)) return e;
    if (int e = res_input(c, mu, ld_mu, N, G, 8, kBufA, &dmu, &up_m)) return e;
    if (int e = ensure(c, kBufC, (size_t)G * 8, &dah)) return e;
    if (int e = ensure(c, kBufD, (size_t)G * 8, &dal)) return e;
    if (int e = ensure(c, kBufE, (size_t)G * 8, &dconv)) return e;
    void* status;
    if (int e = ensure(c, kBufStatus, (size_t)G * sizeof(int), &status)) return e;
    Pipe pp;
    if (int e = vec_h2d(c, dah, alpha_hat, (size_t)G * 8)) return e;
    if (int e = pipe_begin(c, G, {up_c ? (const void*)counts : nullptr, up_m ? (const void*)mu : nullptr}, &pp)) return e;
    for (int b = 0; b < pp.nb; ++b) {
        const int g0 = pp.g0(b), gb = pp.gb(b);
        if (up_c)
            if (int e = cols_h2d(c, pp, b, dc, G, counts, ld, N, 8)) return e;
        if (up_m)
            if (int e = cols_h2d(c, pp, b, dmu, G, mu, ld_mu, N, 8)) return e;
        if (int e = alpha_mle_op(c, pp.cfg_for(b, N), d->d, (const int64_t*)dc + g0, G, gb, (const double*)dmu + g0, G, (const double*)dah + g0,
                                 min_disp, max_disp, prior_disp_var, nullptr, cr_reg, prior_reg, (double*)dal + g0, (double*)dconv + g0,
                                 (int*)status + g0))
            return e;
    }
    if (int e = pipe_join(c, pp)) return e;
    if (int e = vec_d2h(c, alpha_out, dal, (size_t)G * 8)) return e;
    if (int e = vec_d2h(c, conv_out, dconv, (size_t)G * 8)) return e;
    return call_end(c, nullptr, {});
}

extern "C" int pdq_wald_test(pdq_ctx* c, const double* X, int N, int p, const double* disp, const double* lfc, const double* mu,
                             int64_t ld_mu, int G, const double* ridge, const double* contrast, double lfc_null, int alt,
                             double* pv_out, double* stat_out, double* se_out) {
    CHECK_CTX(c);
    if (!X || !disp || !lfc || !mu || !ridge || !contrast || !pv_out || !stat_out || !se_out || N <= 0 || G <= 0 || ld_mu < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_wald_test: bad arguments");
    if (int e = design_width(c, p)) return e;
    if (int e = check_alt(c, alt, "pdq_wald_test: unknown alternative")) return e;
    pdq_design* d;
    if (int e = cached_design(c, X, nullptr, N, p, &d)) return e;
    void *dmu, *ddisp, *dlfc, *dp, *ds, *dse;
    res_begin(c);
    bool up_m;
    if (int e = res_input(c, mu, ld_mu, N, G, 8, kBufA, &dmu, &up_m)) return e;
    if (int e = ensure(c, kBufC, (size_t)G * 8, &ddisp)) return e;
    if (int e = ensure(c, kBufD, (size_t)G * p * 8, &dlfc)) return e;
    if (int e = ensure(c, kBufE, (size_t)G * 8, &dp)) return e;
    if (int e = ensure(c, kBufF, (size_t)G * 8, &ds)) return e;
    if (int e = ensure(c, kBufG, (size_t)G * 8, &dse)) return e;
    Pipe pp;
    if (int e = vec_h2d(c, ddisp, disp, (size_t)G * 8)) return e;
    if (int e = vec_h2d(c, dlfc, lfc, (size_t)G * p * 8)) return e;
    if (int e = pipe_begin(c, G, {up_m ? (const void*)mu : nullptr}, &pp)) return e;
    for (int b = 0; b < pp.nb; ++b) {
        const int g0 = pp.g0(b), gb = pp.gb(b);
        if (up_m)
            if (int e = cols_h2d(c, pp, b, dmu, G, mu, ld_mu, N, 8)) return e;
        if (int e = done(c, launch_wald(pp.cfg_for(b, N), d->d, (const double*)ddisp + g0, (const double*)dlfc + (size_t)g0 * p,
                                        (const double*)dmu + g0, G, gb, ridge, contrast, lfc_null, alt, (double*)dp + g0, (double*)ds + g0,
                                        (double*)dse + g0), "wald_test"))
            return e;
    }
    if (int e = pipe_join(c, pp)) return e;
    if (int e = vec_d2h(c, pv_out, dp, (size_t)G * 8)) return e;
    if (int e = vec_d2h(c, stat_out, ds, (size_t)G * 8)) return e;
    if (int e = vec_d2h(c, se_out, dse, (size_t)G * 8)) return e;
    return call_end(c, nullptr, {});
}

// The test reads G x (p + 1) numbers instead of an (N, G) mu; the (K, G) outputs are the large transfer, so with page-locked
// outputs they leave block by block through the gene-block pipeline while the next block computes.
extern "C" int pdq_wald_contrasts(pdq_ctx* c, const double* X, const double* sf, int N, int p, const double* disp, const double* lfc,
                                  int G, const double* ridge, int K, const double* contrasts, const double* lfc_null, const int* alt,
                                  double* pv_out, double* stat_out, double* se_out, int64_t ld_out) {
    CHECK_CTX(c);
    if (!X || !sf || !disp || !lfc || !ridge || !contrasts || !lfc_null || !alt || !pv_out || !stat_out || !se_out || N <= 0 || p <= 0 ||
        G <= 0 || K <= 0 || ld_out < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_wald_contrasts: bad arguments");
    if (int e = design_width(c, p, false, "pdq_wald_contrasts: ")) return e;
    std::vector<double> tab((size_t)K * (p + 2));
    if (const int k = wald_contrast_table(K, p, contrasts, lfc_null, alt, tab.data()); k >= 0)
        return fail(c, PDQ_ERR_INVALID, "pdq_wald_contrasts: unknown alternative %d (contrast %d)", alt[k], k);
    pdq_design* d;
    if (int e = cached_design(c, X, sf, N, p, &d)) return e;
    const size_t kg = (size_t)K * G;
    void *ddisp, *dlfc, *dtab, *dp, *ds, *dse;
    if (int e = ensure(c, kBufC, (size_t)G * 8, &ddisp)) return e;
    if (int e = ensure(c, kBufD, (size_t)G * p * 8, &dlfc)) return e;
    if (int e = ensure(c, kBufMisc, tab.size() * 8, &dtab)) return e;
    if (int e = ensure(c, kBufA, kg * 8, &dp)) return e;
    if (int e = ensure(c, kBufB, kg * 8, &ds)) return e;
    if (int e = ensure(c, kBufG, kg * 8, &dse)) return e;
    Pipe pp;
    if (int e = vec_h2d(c, ddisp, disp, (size_t)G * 8)) return e;
    if (int e = vec_h2d(c, dlfc, lfc, (size_t)G * p * 8)) return e;
    if (int e = vec_h2d(c, dtab, tab.data(), tab.size() * 8)) return e;
    if (int e = pipe_begin(c, G, {pv_out, stat_out, se_out}, &pp)) return e;
    double* outs[3] = {pv_out, stat_out, se_out};
    void* douts[3] = {dp, ds, dse};
    for (int b = 0; b < pp.nb; ++b) {
        const int g0 = pp.g0(b), gb = pp.gb(b);
        if (int e = done(c, launch_wald_contrasts(pp.cfg_for(b, N), d->d, (const double*)ddisp + g0, (const double*)dlfc + (size_t)g0 * p,
                                                  gb, ridge, K, (const double*)dtab, (double*)dp + g0, (double*)ds + g0, (double*)dse + g0, G),
                         "wald_contrasts"))
            return e;
        for (int i = 0; i < 3; ++i)
            if (int e = cols_d2h(c, pp, b, outs[i], ld_out, douts[i], G, K, 8)) return e;
    }
    return call_end(c, &pp, {});
}

extern "C" int pdq_fit_rough_dispersions(pdq_ctx* c, const double* normed, int64_t ld, int N, int G, const double* X, int p,
                                         double* alpha_out) {
    CHECK_CTX(c);
    if (!normed || !X || !alpha_out || N <= 0 || G <= 0 || ld < G) return fail(c, PDQ_ERR_INVALID, "pdq_fit_rough_dispersions: bad arguments");
    if (int e = check_not_square(c, N, p)) return e;
    pdq_design* d;
    if (int e = cached_design(c, X, nullptr, N, p, &d)) return e;
    void *dn, *da;
    res_begin(c);
    bool up_n;
    if (int e = res_input(c, normed, ld, N, G, 8, kBufA, &dn, &up_n)) return e;
    if (int e = ensure(c, kBufC, (size_t)G * 8, &da)) return e;
    if (up_n)
        if (int e = h2d_2d(c, dn, normed, ld, N, G, 8)) return e;
    if (int e = done(c, launch_rough(cfg(c, G, N), d->d, (const double*)dn, G, G, (double*)da), "fit_rough_dispersions")) return e;
    CU(c, cudaMemcpyAsync(alpha_out, da, (size_t)G * 8, cudaMemcpyDeviceToHost, c->stream));
    return call_end(c, nullptr, {});
}

extern "C" int pdq_fit_moments_dispersions(pdq_ctx* c, const double* normed, int64_t ld, int N, int G, const double* sf,
                                           double* alpha_out, double* all_zero_out) {
    CHECK_CTX(c);
    if (!normed || !sf || !alpha_out || !all_zero_out || N <= 0 || G <= 0 || ld < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_fit_moments_dispersions: bad arguments");
    // a one-column design carries the size factors (the moments estimator does not use X)
    std::vector<double> ones((size_t)N, 1.0);
    pdq_design* d;
    if (int e = cached_design(c, ones.data(), sf, N, 1, &d)) return e;
    void *dn, *da, *dz;
    res_begin(c);
    bool up_n;
    if (int e = res_input(c, normed, ld, N, G, 8, kBufA, &dn, &up_n)) return e;
    if (int e = ensure(c, kBufC, (size_t)G * 8, &da)) return e;
    if (int e = ensure(c, kBufE, (size_t)G * 8, &dz)) return e;
    if (up_n)
        if (int e = h2d_2d(c, dn, normed, ld, N, G, 8)) return e;
    if (int e = done(c, launch_moments(cfg(c, G, N), d->d, (const double*)dn, G, G, (double*)da, (double*)dz), "fit_moments_dispersions")) return e;
    CU(c, cudaMemcpyAsync(alpha_out, da, (size_t)G * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaMemcpyAsync(all_zero_out, dz, (size_t)G * 8, cudaMemcpyDeviceToHost, c->stream));
    return call_end(c, nullptr, {});
}

extern "C" int pdq_calculate_cooks(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, const double* sf, const double* X, int p,
                                   const double* mu, const double* hat, int64_t ld2, double cutoff, double* cooks_out, double* robust_disp_out,
                                   double* outlier_out, double* replaced_out) {
    CHECK_CTX(c);
    if (!counts || !sf || !X || !mu || !hat || !robust_disp_out || !outlier_out || !replaced_out || N <= 0 || G <= 0 || ld < G || ld2 < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_calculate_cooks: bad arguments");
    pdq_design* d;
    if (int e = cached_design(c, X, sf, N, p, &d)) return e;
    const size_t ng = (size_t)N * G;
    void *dc, *dmu, *dhat, *dck = nullptr, *dd, *dout, *drep;
    res_begin(c);
    bool up_c, up_m, up_h;
    if (int e = res_input(c, counts, ld, N, G, 8, kBufCounts, &dc, &up_c)) return e;
    if (int e = res_input(c, mu, ld2, N, G, 8, kBufA, &dmu, &up_m)) return e;
    if (int e = res_input(c, hat, ld2, N, G, 8, kBufB, &dhat, &up_h)) return e;
    if (cooks_out)
        if (int e = ensure(c, kBufRes, ng * 8, &dck)) return e;
    if (int e = ensure(c, kBufC, (size_t)G * 8, &dd)) return e;
    if (int e = ensure(c, kBufE, (size_t)G * 8, &dout)) return e;
    if (int e = ensure(c, kBufF, (size_t)G * 8, &drep)) return e;
    if (up_c)
        if (int e = h2d_2d(c, dc, counts, ld, N, G, 8)) return e;
    if (up_m)
        if (int e = h2d_2d(c, dmu, mu, ld2, N, G, 8)) return e;
    if (up_h)
        if (int e = h2d_2d(c, dhat, hat, ld2, N, G, 8)) return e;
    if (int e = pdq_cooks_dev(c, d, (const int64_t*)dc, G, G, (const double*)dmu, (const double*)dhat, G, cutoff, (double*)dck, G, (double*)dd,
                              (double*)dout, (double*)drep))
        return e;
    if (cooks_out)
        if (int e = copy_d2h(c, cooks_out, dck, ng * 8)) return e;
    CU(c, cudaMemcpyAsync(robust_disp_out, dd, (size_t)G * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaMemcpyAsync(outlier_out, dout, (size_t)G * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaMemcpyAsync(replaced_out, drep, (size_t)G * 8, cudaMemcpyDeviceToHost, c->stream));
    return call_end(c, nullptr, {});
}

extern "C" int pdq_lfc_shrink_nbinom_glm(pdq_ctx* c, const double* X, const int64_t* counts, int64_t ld, int N, int G, int p, const double* size,
                                         const double* offset, double prior_no_shrink_scale, double prior_scale, int shrink_index,
                                         double* lfcs_out, double* inv_hessians_out, double* conv_out, int* n_grid) {
    CHECK_CTX(c);
    if (!X || !counts || !size || !offset || !lfcs_out || !inv_hessians_out || !conv_out || N <= 0 || G <= 0 || ld < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_lfc_shrink_nbinom_glm: bad arguments");
    if (int e = design_width(c, p)) return e;
    if (int e = design_width(c, p, true)) return e;
    if (int e = check_shrink(c, p, shrink_index, prior_no_shrink_scale, prior_scale)) return e;
    pdq_design* d;  // the kernel reads the offsets from the log-size-factor row of the design pack
    if (int e = cached_design(c, X, offset, N, p, &d, true)) return e;
    void *dc, *dsize, *dbeta, *dih, *dconv, *status;
    res_begin(c);
    bool up_c;
    if (int e = res_input(c, counts, ld, N, G, 8, kBufCounts, &dc, &up_c)) return e;
    if (int e = ensure(c, kBufC, (size_t)G * 8, &dsize)) return e;
    if (int e = ensure(c, kBufD, (size_t)G * p * 8, &dbeta)) return e;
    if (int e = ensure(c, kBufA, (size_t)G * p * p * 8, &dih)) return e;
    if (int e = ensure(c, kBufE, (size_t)G * 8, &dconv)) return e;
    if (int e = ensure(c, kBufStatus, (size_t)G * sizeof(int), &status)) return e;
    if (up_c)
        if (int e = h2d_2d(c, dc, counts, ld, N, G, 8)) return e;
    CU(c, cudaMemcpyAsync(dsize, size, (size_t)G * 8, cudaMemcpyHostToDevice, c->stream));
    // the one launch site of apeGLM shrinkage, whose checks (passed above, before anything was staged) it runs again
    if (int e = pdq_lfc_shrink_dev(c, d, (const int64_t*)dc, G, G, (const double*)dsize, prior_no_shrink_scale, prior_scale, shrink_index,
                                   (double*)dbeta, (double*)dih, (double*)dconv, (int*)status))
        return e;
    CU(c, cudaMemcpyAsync(lfcs_out, dbeta, (size_t)G * p * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaMemcpyAsync(inv_hessians_out, dih, (size_t)G * p * p * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaMemcpyAsync(conv_out, dconv, (size_t)G * 8, cudaMemcpyDeviceToHost, c->stream));
    std::vector<int> st;
    if (n_grid) {
        st.resize((size_t)G);
        CU(c, cudaMemcpyAsync(st.data(), status, (size_t)G * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    }
    if (int e = call_end(c, nullptr, {})) return e;
    if (n_grid) {
        *n_grid = 0;
        for (int v : st) *n_grid += (v != 0);
    }
    return PDQ_OK;
}

extern "C" int pdq_size_factors(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, double* sf_out, double* logmeans_out) {
    CHECK_CTX(c);
    if (!counts || !sf_out || N <= 0 || G <= 0 || ld < G) return fail(c, PDQ_ERR_INVALID, "pdq_size_factors: bad arguments");
    void *dc, *dsf, *dlm = nullptr;
    res_begin(c);
    bool up_c;
    if (int e = res_input(c, counts, ld, N, G, 8, kBufCounts, &dc, &up_c)) return e;
    if (int e = ensure(c, kBufE, (size_t)N * 8, &dsf)) return e;
    if (logmeans_out)
        if (int e = ensure(c, kBufG, (size_t)G * 8, &dlm)) return e;
    if (up_c)
        if (int e = h2d_2d(c, dc, counts, ld, N, G, 8)) return e;
    if (int e = pdq_size_factors_dev(c, (const int64_t*)dc, G, N, G, (double*)dsf, (double*)dlm)) return e;
    CU(c, cudaMemcpyAsync(sf_out, dsf, (size_t)N * 8, cudaMemcpyDeviceToHost, c->stream));
    if (logmeans_out) CU(c, cudaMemcpyAsync(logmeans_out, dlm, (size_t)G * 8, cudaMemcpyDeviceToHost, c->stream));
    return call_end(c, nullptr, {});
}

extern "C" int pdq_size_factors_ex(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, int kind, const uint8_t* control,
                                   double* sf_out, double* logmeans_out) {
    CHECK_CTX(c);
    if (int e = sf_ex_check(c, counts, sf_out, ld, N, G, kind, "pdq_size_factors_ex")) return e;
    void *dc, *dsf, *dlm = nullptr, *dctl = nullptr;
    res_begin(c);
    bool up_c;
    if (int e = res_input(c, counts, ld, N, G, 8, kBufCounts, &dc, &up_c)) return e;
    if (int e = ensure(c, kBufE, (size_t)N * 8, &dsf)) return e;
    if (logmeans_out)
        if (int e = ensure(c, kBufG, (size_t)G * 8, &dlm)) return e;
    if (control)
        if (int e = ensure(c, kBufKeep, (size_t)G, &dctl)) return e;
    if (up_c)
        if (int e = h2d_2d(c, dc, counts, ld, N, G, 8)) return e;
    if (control)
        if (int e = vec_h2d(c, dctl, control, (size_t)G)) return e;
    if (int e = pdq_size_factors_ex_dev(c, (const int64_t*)dc, G, N, G, kind, (const uint8_t*)dctl, (double*)dsf, (double*)dlm)) return e;
    CU(c, cudaMemcpyAsync(sf_out, dsf, (size_t)N * 8, cudaMemcpyDeviceToHost, c->stream));
    if (logmeans_out) CU(c, cudaMemcpyAsync(logmeans_out, dlm, (size_t)G * 8, cudaMemcpyDeviceToHost, c->stream));
    return call_end(c, nullptr, {});
}

extern "C" int pdq_size_factors_from_logmeans(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, const double* logmeans,
                                              double* sf_out) {
    CHECK_CTX(c);
    if (!counts || !logmeans || !sf_out || N <= 0 || G <= 0 || ld < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_size_factors_from_logmeans: bad arguments");
    void *dc, *dsf, *dlm;
    res_begin(c);
    bool up_c;
    if (int e = res_input(c, counts, ld, N, G, 8, kBufCounts, &dc, &up_c)) return e;
    if (int e = ensure(c, kBufE, (size_t)N * 8, &dsf)) return e;
    if (int e = ensure(c, kBufG, (size_t)G * 8, &dlm)) return e;
    if (up_c)
        if (int e = h2d_2d(c, dc, counts, ld, N, G, 8)) return e;
    if (int e = vec_h2d(c, dlm, logmeans, (size_t)G * 8)) return e;
    if (int e = pdq_size_factors_from_logmeans_dev(c, (const int64_t*)dc, G, N, G, (const double*)dlm, (double*)dsf)) return e;
    CU(c, cudaMemcpyAsync(sf_out, dsf, (size_t)N * 8, cudaMemcpyDeviceToHost, c->stream));
    return call_end(c, nullptr, {});
}

// counts through the residency cache (after the fit calls of vst_fit they are on the device already), the (N, G) result back
// through the page-locked staging ring, in gene blocks overlapping the download with the next block's transform
extern "C" int pdq_vst_transform(pdq_ctx* c, const int64_t* counts, int64_t ld, int N, int G, const double* size_factors, int kind,
                                 double c0, double c1, double* out, int64_t ld_out) {
    CHECK_CTX(c);
    if (int e = vst_check(c, counts, size_factors, out, ld, N, G, kind, c0, ld_out, "pdq_vst_transform")) return e;
    void *dc, *dsf, *dout;
    res_begin(c);
    bool up_c;
    if (int e = res_input(c, counts, ld, N, G, 8, kBufCounts, &dc, &up_c)) return e;
    if (int e = ensure(c, kBufE, (size_t)N * 8, &dsf)) return e;
    if (int e = ensure(c, kBufA, (size_t)N * G * 8, &dout)) return e;
    if (int e = vec_h2d(c, dsf, size_factors, (size_t)N * 8)) return e;
    Pipe pp;
    if (int e = pipe_begin(c, G, {up_c ? (const void*)counts : nullptr, out}, &pp)) return e;
    for (int b = 0; b < pp.nb; ++b) {
        if (up_c)
            if (int e = cols_h2d(c, pp, b, dc, G, counts, ld, N, 8)) return e;
        if (int e = done(c, launch_vst_transform(pp.cfg_for(b, N), (const int64_t*)dc + pp.g0(b), G, N, pp.gb(b), (const double*)dsf, kind,
                                                 c0, c1, (double*)dout + pp.g0(b), G),
                         "vst_transform"))
            return e;
        if (int e = cols_d2h(c, pp, b, out, ld_out, dout, G, N, 8)) return e;
    }
    return call_end(c, &pp, {});
}

extern "C" int pdq_dispersion_trend_gamma_glm(pdq_ctx* c, const double* cov, const double* targets, size_t n, double* coeffs_out,
                                              double* pred_out, int* converged_out) {
    CHECK_CTX(c);
    if (!cov || !targets || !coeffs_out || !pred_out || !converged_out || n == 0)
        return fail(c, PDQ_ERR_INVALID, "pdq_dispersion_trend_gamma_glm: bad arguments");
    void *dx, *dt, *scratch, *dout;
    if (int e = ensure(c, kBufC, n * 8, &dx)) return e;
    if (int e = ensure(c, kBufD, n * 8, &dt)) return e;
    if (int e = ensure(c, kBufRes, 3 * n * 8, &scratch)) return e;
    if (int e = ensure(c, kBufMisc, 256, &dout)) return e;
    CU(c, cudaMemcpyAsync(dx, cov, n * 8, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(dt, targets, n * 8, cudaMemcpyHostToDevice, c->stream));
    LaunchCfg lc{c->stream, 0, c->prop.multiProcessorCount, c->tickets, c->debug, c->grid_scratch};
    const double inf = 1.0 / 0.0;
    if (int e = done(c, launch_trend_fit(lc, (const double*)dx, (const double*)dt, (double*)scratch, n, 0, -inf, inf, 0, 0.0, 0.0, 0, (double*)dout),
                     "dispersion_trend_gamma_glm"))
        return e;
    double out[16];
    CU(c, cudaMemcpyAsync(out, dout, sizeof out, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    coeffs_out[0] = out[0];
    coeffs_out[1] = out[1];
    *converged_out = out[7] != 0.0;  // the reference's flag is L-BFGS-B's `success`; ours: the iteration converged
    for (size_t i = 0; i < n; ++i) pred_out[i] = out[0] + out[1] * cov[i];
    return PDQ_OK;
}

// Trend + prior in one launch with host vectors: the orchestrator's whole `fit_dispersion_trend` loop (dds.py:1199-1275) and
// `fit_dispersion_prior` (dds.py:840-884) -- what pdq_trend_fit_dev does for the resident pipeline.  out16 = TrendOut record.
extern "C" int pdq_trend_prior(pdq_ctx* c, const double* means, const double* genewise, size_t n, double min_disp, double max_disp,
                               double trigamma_c, double* out16, double* fitted_out) {
    CHECK_CTX(c);
    if (!means || !genewise || !out16 || n == 0) return fail(c, PDQ_ERR_INVALID, "pdq_trend_prior: bad arguments");
    void *dm, *dg, *df, *dout;
    if (int e = ensure(c, kBufC, n * 8, &dm)) return e;
    if (int e = ensure(c, kBufD, n * 8, &dg)) return e;
    if (int e = ensure(c, kBufF, n * 8, &df)) return e;
    if (int e = ensure(c, kBufMisc, 256, &dout)) return e;
    CU(c, cudaMemcpyAsync(dm, means, n * 8, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(dg, genewise, n * 8, cudaMemcpyHostToDevice, c->stream));
    if (int e = pdq_trend_fit_dev(c, (const double*)dm, (const double*)dg, n, min_disp, max_disp, trigamma_c, (double*)dout,
                                  fitted_out ? (double*)df : nullptr))
        return e;
    CU(c, cudaMemcpyAsync(out16, dout, 16 * 8, cudaMemcpyDeviceToHost, c->stream));
    if (fitted_out) CU(c, cudaMemcpyAsync(fitted_out, df, n * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return PDQ_OK;
}

// --------------------------------------------------------------------------------------------- multiple testing (ds.py:486-542)
// Host vectors in and out; the device scratch is one context buffer of its own (pdq_padj.cu, padj_layout).
static int padj_begin(pdq_ctx* c, const double* base_mean, int G, const double* pvalues, int64_t ld, int K, int n_theta, PadjScratch* s) {
    void* base;
    if (int e = ensure(c, kBufPadj, padj_layout(G, K, n_theta, nullptr, s), &base)) return e;
    padj_layout(G, K, n_theta, base, s);
    if (int e = vec_h2d(c, s->bm, base_mean, (size_t)G * 8)) return e;
    return h2d_2d(c, s->keys_in, pvalues, ld, K, G, 8);
}

static int padj_end(pdq_ctx* c, const PadjScratch& s, int K, const char* what) {
    int bad = 0;
    CU(c, cudaMemcpyAsync(&bad, s.counters + K, sizeof bad, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (bad) return fail(c, PDQ_ERR_INVALID, "%s: %d p-value(s) outside [0, 1]", what, bad);
    return PDQ_OK;
}

extern "C" int pdq_padj_rejections(pdq_ctx* c, const double* base_mean, int G, const double* pvalues, int64_t ld, int K,
                                   const double* theta, int n_theta, double alpha, double* cutoffs_out, int* num_rej_out) {
    CHECK_CTX(c);
    if (!base_mean || !pvalues || !theta || !cutoffs_out || !num_rej_out || G <= 0 || K <= 0 || ld < G || n_theta <= 0 ||
        n_theta > kPadjMaxTheta)
        return fail(c, PDQ_ERR_INVALID, "pdq_padj_rejections: bad arguments (G=%d, K=%d, ld=%lld, n_theta=%d)", G, K, (long long)ld,
                    n_theta);
    PadjScratch s;
    if (int e = padj_begin(c, base_mean, G, pvalues, ld, K, n_theta, &s)) return e;
    if (int e = vec_h2d(c, s.theta, theta, (size_t)n_theta * 8)) return e;
    if (int e = done(c, launch_padj_rejections(c->stream, s, G, K, n_theta, alpha), "padj_rejections")) return e;
    if (int e = vec_d2h(c, cutoffs_out, s.cutoffs, (size_t)n_theta * 8)) return e;
    if (int e = vec_d2h(c, num_rej_out, s.num_rej, (size_t)K * n_theta * sizeof(int))) return e;
    return padj_end(c, s, K, "pdq_padj_rejections");
}

extern "C" int pdq_padj_bh(pdq_ctx* c, const double* base_mean, int G, const double* pvalues, int64_t ld, int K, const double* cutoff,
                           double* padj_out, int64_t ld_out) {
    CHECK_CTX(c);
    if (!base_mean || !pvalues || !cutoff || !padj_out || G <= 0 || K <= 0 || ld < G || ld_out < G)
        return fail(c, PDQ_ERR_INVALID, "pdq_padj_bh: bad arguments (G=%d, K=%d, ld=%lld, ld_out=%lld)", G, K, (long long)ld,
                    (long long)ld_out);
    PadjScratch s;
    if (int e = padj_begin(c, base_mean, G, pvalues, ld, K, 1, &s)) return e;
    if (int e = vec_h2d(c, s.row_cutoff, cutoff, (size_t)K * 8)) return e;
    double* d_out = (double*)s.keys_in;  // free once the rows are sorted
    if (int e = done(c, launch_padj_bh(c->stream, s, G, K, d_out, G), "padj_bh")) return e;
    if (ld_out == G) {
        if (int e = copy_d2h(c, padj_out, d_out, (size_t)K * G * 8)) return e;
    } else {
        CU(c, cudaMemcpy2DAsync(padj_out, (size_t)ld_out * 8, d_out, (size_t)G * 8, (size_t)G * 8, K, cudaMemcpyDeviceToHost, c->stream));
    }
    return padj_end(c, s, K, "pdq_padj_bh");
}

// --------------------------------------------------------------------------------------------- NCCL gene-shard exchange
static int nccl_load(pdq_ctx* c) {
    if (c->nccl.handle) return 0;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
        c->nccl.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (c->nccl.handle) break;
    }
    if (!c->nccl.handle) return fail(c, PDQ_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
    auto sym = [&](const char* s) { return dlsym(c->nccl.handle, s); };
    c->nccl.GetUniqueId = (decltype(c->nccl.GetUniqueId))sym("ncclGetUniqueId");
    c->nccl.CommInitRank = (decltype(c->nccl.CommInitRank))sym("ncclCommInitRank");
    c->nccl.AllGather = (decltype(c->nccl.AllGather))sym("ncclAllGather");
    c->nccl.CommDestroy = (decltype(c->nccl.CommDestroy))sym("ncclCommDestroy");
    c->nccl.GetErrorString = (decltype(c->nccl.GetErrorString))sym("ncclGetErrorString");
    c->nccl.GroupStart = (decltype(c->nccl.GroupStart))sym("ncclGroupStart");
    c->nccl.GroupEnd = (decltype(c->nccl.GroupEnd))sym("ncclGroupEnd");
    if (!c->nccl.GetUniqueId || !c->nccl.CommInitRank || !c->nccl.AllGather || !c->nccl.CommDestroy || !c->nccl.GroupStart ||
        !c->nccl.GroupEnd)
        return fail(c, PDQ_ERR_NCCL, "libnccl is missing a required symbol");
    return 0;
}

static int nccl_fail(pdq_ctx* c, ncclResult_t r, const char* what) {
    return fail(c, PDQ_ERR_NCCL, "%s failed: %s", what, c->nccl.GetErrorString ? c->nccl.GetErrorString(r) : "nccl error");
}

extern "C" int pdq_comm_unique_id(pdq_ctx* c, void* id_out) {
    CHECK_CTX(c);
    if (!id_out) return PDQ_ERR_INVALID;
    if (int e = nccl_load(c)) return e;
    ncclUniqueId id;
    ncclResult_t r = c->nccl.GetUniqueId(&id);
    if (r != 0) return nccl_fail(c, r, "ncclGetUniqueId");
    static_assert(sizeof(id) == PDQ_UNIQUE_ID_BYTES, "ncclUniqueId size");
    memcpy(id_out, &id, sizeof id);
    return PDQ_OK;
}

extern "C" int pdq_comm_init(pdq_ctx* c, const void* id, int world, int rank) {
    CHECK_CTX(c);
    if (!id || world < 1 || rank < 0 || rank >= world) return fail(c, PDQ_ERR_INVALID, "pdq_comm_init: bad arguments");
    if (int e = nccl_load(c)) return e;
    ncclUniqueId uid;
    memcpy(&uid, id, sizeof uid);
    ncclResult_t r = c->nccl.CommInitRank(&c->comm, world, uid, rank);
    if (r != 0) return nccl_fail(c, r, "ncclCommInitRank");
    c->world = world;
    c->rank = rank;
    return PDQ_OK;
}

extern "C" int pdq_allgather_f64_dev(pdq_ctx* c, const double* send, double* recv, size_t count) {
    CHECK_CTX(c);
    if (!send || !recv) return PDQ_ERR_INVALID;
    if (!c->comm) {  // single rank: the gather is a copy
        if (send != recv) CU(c, cudaMemcpyAsync(recv, send, count * 8, cudaMemcpyDeviceToDevice, c->stream));
        return PDQ_OK;
    }
    ncclResult_t r = c->nccl.AllGather(send, recv, count, kNcclFloat64, c->comm, c->stream);
    if (r != 0) return nccl_fail(c, r, "ncclAllGather");
    return PDQ_OK;
}

// k equal-count all-gathers issued as ONE NCCL group (one fused launch on the stream): the exchange of the per-gene vectors the
// trend / prior step needs from every gene shard, and the end-of-call exchange of the result tables
extern "C" int pdq_allgather_multi_f64_dev(pdq_ctx* c, int k, const double* const* send, double* const* recv, size_t count) {
    CHECK_CTX(c);
    if (k < 1 || k > 16 || !send || !recv) return fail(c, PDQ_ERR_INVALID, "pdq_allgather_multi_f64_dev: bad arguments");
    for (int i = 0; i < k; ++i)
        if (!send[i] || !recv[i]) return fail(c, PDQ_ERR_INVALID, "pdq_allgather_multi_f64_dev: null buffer");
    if (!c->comm) {  // single rank: the gathers are copies
        for (int i = 0; i < k; ++i)
            if (send[i] != recv[i]) CU(c, cudaMemcpyAsync(recv[i], send[i], count * 8, cudaMemcpyDeviceToDevice, c->stream));
        return PDQ_OK;
    }
    ncclResult_t r = c->nccl.GroupStart();
    if (r != 0) return nccl_fail(c, r, "ncclGroupStart");
    for (int i = 0; i < k; ++i) {
        r = c->nccl.AllGather(send[i], recv[i], count, kNcclFloat64, c->comm, c->stream);
        if (r != 0) {
            c->nccl.GroupEnd();
            return nccl_fail(c, r, "ncclAllGather");
        }
    }
    r = c->nccl.GroupEnd();
    if (r != 0) return nccl_fail(c, r, "ncclGroupEnd");
    return PDQ_OK;
}

// --------------------------------------------------------------------------------------------- peer-memory gene-shard exchange
// The same two exchanges without NCCL: every rank owns one "window" (a cudaMalloc block exported with CUDA IPC and mapped by all
// peers of the node).  ONE kernel per exchange reads the rank's segment once and stores it into the same place of EVERY rank's
// window over NVLink / NVSwitch (plain peer stores), then signals the peers and waits for theirs: copy + barrier in one launch,
// capturable in the pass's CUDA graph.  Window layout: 4096 bytes of control words, data behind.
//   control: word 0 = number of exchanges this rank has completed, word 1 = finished blocks of the running push (both local);
//   byte 128 * (1 + r) = arrival counter of rank r: the last block of r's push kernel adds 1 after all of r's stores are fenced
//   system-wide.
static constexpr int kPeerMaxWorld = 16, kPeerThreads = 512;
static constexpr size_t kPeerCtrlBytes = 4096;

struct pdq_peer_group {
    int world = 1, rank = 0;
    void* base[kPeerMaxWorld] = {};      // every rank's window as mapped in THIS process (base[rank] = the own allocation)
    unsigned long long* err_host = nullptr;  // mapped page-locked word: non-zero after a push kernel gave up waiting
    unsigned long long* err_dev = nullptr;
};

struct PeerPushArgs {
    char* base[kPeerMaxWorld];
    int world, rank, k;
    const double* send[4];
    unsigned long long recv_off[4];  // byte offset of the gathered vector in the window (behind the control words)
    unsigned long long count;        // doubles per rank and segment
    unsigned long long* err;
    unsigned long long timeout_ns;
};

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__global__ void __launch_bounds__(kPeerThreads) k_peer_push(const PeerPushArgs a) {
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
    for (int s = 0; s < a.k; ++s) {
        const double* src = a.send[s];
        const size_t dst_off = kPeerCtrlBytes + a.recv_off[s] + (size_t)a.rank * a.count * 8;
        const bool vec = (a.count % 2 == 0) && (((uintptr_t)src | dst_off) % 16 == 0);
        if (vec) {
            const double2* src2 = reinterpret_cast<const double2*>(src);
            for (size_t i = tid; i < a.count / 2; i += nth) {
                const double2 v = src2[i];
                for (int q = 0; q < a.world; ++q) {  // own window last: the remote stores leave first
                    const int r = (a.rank + 1 + q) % a.world;
                    reinterpret_cast<double2*>(a.base[r] + dst_off)[i] = v;
                }
            }
        } else {
            for (size_t i = tid; i < a.count; i += nth) {
                const double v = src[i];
                for (int q = 0; q < a.world; ++q) {
                    const int r = (a.rank + 1 + q) % a.world;
                    reinterpret_cast<double*>(a.base[r] + dst_off)[i] = v;
                }
            }
        }
    }
    // the LAST block of this rank to finish its stores signals the peers (one arrival per rank and exchange, whatever the grid)
    __shared__ int last;
    unsigned long long* ctrl = reinterpret_cast<unsigned long long*>(a.base[a.rank]);
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        const unsigned long long done = atomicAdd(&ctrl[1], 1ULL);
        last = (done == gridDim.x - 1);
        if (last) {
            ctrl[1] = 0;
            __threadfence_system();
            for (int q = 1; q < a.world; ++q) {
                const int r = (a.rank + q) % a.world;
                atomicAdd_system(reinterpret_cast<unsigned long long*>(a.base[r] + 128 * (1 + a.rank)), 1ULL);
            }
        }
    }
    __syncthreads();
    if (!last) return;
    // ... and waits until every peer's segments of the same exchange have arrived here
    const unsigned long long target = ctrl[0] + 1;
    if ((int)threadIdx.x < a.world && (int)threadIdx.x != a.rank) {
        const unsigned long long* flag = reinterpret_cast<const unsigned long long*>(a.base[a.rank] + 128 * (1 + threadIdx.x));
        const unsigned long long t0 = global_timer_ns();
        while (ld_acquire_sys(flag) < target) {
            if (global_timer_ns() - t0 > a.timeout_ns) {  // a peer never arrived: report instead of hanging the GPU
                *a.err = 1ULL + threadIdx.x;
                __threadfence_system();
                break;
            }
            __nanosleep(64);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) ctrl[0] = target;
}

extern "C" int pdq_peer_window_alloc(pdq_ctx* c, size_t data_bytes, void** window_out, void** data_out, void* handle_out) {
    CHECK_CTX(c);
    if (!window_out || !data_out || !handle_out) return fail(c, PDQ_ERR_INVALID, "pdq_peer_window_alloc: bad arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == PDQ_PEER_HANDLE_BYTES, "cudaIpcMemHandle_t size");
    void* w = nullptr;
    CU(c, cudaMalloc(&w, kPeerCtrlBytes + data_bytes));
    CU(c, cudaMemsetAsync(w, 0, kPeerCtrlBytes, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    cudaIpcMemHandle_t hd;
    cudaError_t e = cudaIpcGetMemHandle(&hd, w);
    if (e != cudaSuccess) {
        cudaFree(w);
        return fail(c, PDQ_ERR_CUDA, "cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    }
    memcpy(handle_out, &hd, sizeof hd);
    *window_out = w;
    *data_out = (char*)w + kPeerCtrlBytes;
    return PDQ_OK;
}

extern "C" int pdq_peer_window_free(pdq_ctx* c, void* window) {
    CHECK_CTX(c);
    if (window) CU(c, cudaFree(window));
    return PDQ_OK;
}

extern "C" int pdq_peer_group_open(pdq_ctx* c, void* own_window, int world, int rank, const void* handles, pdq_peer_group** out) {
    CHECK_CTX(c);
    if (!own_window || !handles || !out || world < 1 || world > kPeerMaxWorld || rank < 0 || rank >= world)
        return fail(c, PDQ_ERR_INVALID, "pdq_peer_group_open: bad arguments (world <= %d)", kPeerMaxWorld);
    pdq_peer_group* g = new pdq_peer_group;
    g->world = world;
    g->rank = rank;
    for (int r = 0; r < world; ++r) {
        if (r == rank) {
            g->base[r] = own_window;
            continue;
        }
        cudaIpcMemHandle_t hd;
        memcpy(&hd, (const char*)handles + (size_t)r * sizeof hd, sizeof hd);
        cudaError_t e = cudaIpcOpenMemHandle(&g->base[r], hd, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
            for (int q = 0; q < r; ++q)
                if (q != rank) cudaIpcCloseMemHandle(g->base[q]);
            delete g;
            cudaGetLastError();
            return fail(c, PDQ_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e));
        }
    }
    cudaError_t e = cudaHostAlloc((void**)&g->err_host, 8, cudaHostAllocMapped);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer((void**)&g->err_dev, g->err_host, 0);
    if (e != cudaSuccess) {
        for (int q = 0; q < world; ++q)
            if (q != rank) cudaIpcCloseMemHandle(g->base[q]);
        delete g;
        return fail(c, PDQ_ERR_CUDA, "cudaHostAlloc(peer status) failed: %s", cudaGetErrorString(e));
    }
    *g->err_host = 0;
    *out = g;
    return PDQ_OK;
}

// k (<= 4) segments of `count` doubles each: segment i of this rank lands at data offset recv_off_bytes[i] + rank * count * 8 of
// EVERY rank's window; returns (on the stream) once all ranks' segments have landed here.  k = 0: barrier only.
extern "C" int pdq_peer_push_dev(pdq_ctx* c, pdq_peer_group* g, int k, const double* const* send, const unsigned long long* recv_off_bytes,
                                 size_t count) {
    CHECK_CTX(c);
    if (!g || k < 0 || k > 4 || (k > 0 && (!send || !recv_off_bytes))) return fail(c, PDQ_ERR_INVALID, "pdq_peer_push_dev: bad arguments");
    PeerPushArgs a{};
    for (int r = 0; r < g->world; ++r) a.base[r] = (char*)g->base[r];
    a.world = g->world;
    a.rank = g->rank;
    a.k = k;
    for (int i = 0; i < k; ++i) {
        if (!send[i] || recv_off_bytes[i] % 8) return fail(c, PDQ_ERR_INVALID, "pdq_peer_push_dev: bad segment");
        a.send[i] = send[i];
        a.recv_off[i] = recv_off_bytes[i];
    }
    a.count = count;
    a.err = g->err_dev;
    static const unsigned long long timeout_ms = getenv("PDQ_PEER_TIMEOUT_MS") ? strtoull(getenv("PDQ_PEER_TIMEOUT_MS"), nullptr, 10) : 30000ULL;
    a.timeout_ns = timeout_ms * 1000000ULL;
    // 64 blocks of 512 threads: enough stores in flight for the NVLink path, and a short tail before the signal (not re-tuned on
    // H100: the multi-GPU path has not been measured there); PDQ_PEER_BLOCKS overrides
    static const int forced = getenv("PDQ_PEER_BLOCKS") ? atoi(getenv("PDQ_PEER_BLOCKS")) : 0;
    const int blocks = forced > 0 ? forced : 64;
    k_peer_push<<<blocks, kPeerThreads, 0, c->stream>>>(a);
    CU(c, cudaGetLastError());
    c->launches += 1;
    return PDQ_OK;
}

// 0 while every exchange completed; 1 + r when a push kernel gave up waiting for rank r (valid after a stream synchronisation)
extern "C" int pdq_peer_status(pdq_ctx* c, pdq_peer_group* g, unsigned long long* status_out) {
    CHECK_CTX(c);
    if (!g || !status_out) return fail(c, PDQ_ERR_INVALID, "pdq_peer_status: bad arguments");
    *status_out = *(volatile unsigned long long*)g->err_host;
    return PDQ_OK;
}

// unmaps the peers' windows (every rank must do so BEFORE any rank frees its own window)
extern "C" int pdq_peer_group_close(pdq_ctx* c, pdq_peer_group* g) {
    CHECK_CTX(c);
    if (!g) return PDQ_OK;
    CU(c, cudaStreamSynchronize(c->stream));
    for (int r = 0; r < g->world; ++r)
        if (r != g->rank && g->base[r]) cudaIpcCloseMemHandle(g->base[r]);
    if (g->err_host) cudaFreeHost(g->err_host);
    delete g;
    return PDQ_OK;
}

extern "C" int pdq_comm_destroy(pdq_ctx* c) {
    CHECK_CTX(c);
    if (c->comm) {
        c->nccl.CommDestroy(c->comm);
        c->comm = nullptr;
    }
    c->world = 1;
    c->rank = 0;
    return PDQ_OK;
}
