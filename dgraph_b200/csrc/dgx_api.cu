// dgx_api.cu -- libdgx.so: C ABI (include/dgx.h) over the sm_90a kernels.
//
// Host responsibilities only: lane (stream + workspace) management, building the
// small task / list descriptor tables the kernels read, host<->device copies for
// the host-pointer entry points.  No set-operation or decode arithmetic runs on
// the CPU here: if CUDA is unavailable every entry point fails with
// DGX_ERR_NODEV / DGX_ERR_CUDA (the cgo shim then stays on the Go path).
#include "../../include/dgx.h"

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <list>
#include <mutex>
#include <numeric>
#include <string>
#include <unordered_map>
#include <vector>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include "decode_kernel.cuh"
#include "filter_kernel.cuh"
#include "filter_pipe.cuh"
#include "merge_kernel.cuh"
#include "merge_multi.cuh"
#include "merge_tile32.cuh"
#include "merge_matrix.cuh"
#include "probe_kernel.cuh"
#include "compressed_kernel.cuh"
#include "list_uids_kernel.cuh"
#include "list_uids_unfiltered_kernel.cuh"
#include "encode_kernel.cuh"
#include "backup_codec_kernel.cuh"
#include "trigram_kernel.cuh"
#include "groupby_kernel.cuh"
#include "recurse_kernel.cuh"
#include "cascade_kernel.cuh"
#include "path_kernel.cuh"
#include "valvar_kernel.cuh"
#include "math_kernel.cuh"
#include "sg_filter_kernel.cuh"
#include "var_order_kernel.cuh"
#include "match_kernel.cuh"
#include "regex_kernel.cuh"
#include "regex_compile.hpp"
#include "compare_kernel.cuh"
#include "pred_order_kernel.cuh"
#include "wire.hpp"
#include "ws_layout.hpp"

using namespace dgx;

// ---------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------
static thread_local std::string g_err;

static int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CK(call)                                                                              \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess)                                                                \
            return fail(e_ == cudaErrorMemoryAllocation ? DGX_ERR_OOM : DGX_ERR_CUDA,         \
                        "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

extern "C" const char* dgx_last_error(void) { return g_err.c_str(); }

// ---------------------------------------------------------------------------
// global state
// ---------------------------------------------------------------------------
struct Stats {
    std::atomic<uint64_t> calls{0}, uids_in{0}, uids_out{0}, h2d{0}, d2h{0}, launches{0};
};
static Stats g_stats;
static std::atomic<uint64_t> g_xm_overflows{0};  // chunks of dgx_*merge_sorted_matrix sorted in global memory
static std::atomic<uint64_t> g_tail_queries{0};  // filter queries whose sparse tail filter_tail_kernel served
static std::mutex g_mu;
static int g_device = -1;
static std::vector<dgx_lane*> g_pool;  // idle lanes for the host-pointer entry points
static std::condition_variable g_pool_cv;
static size_t g_lanes_out = 0;     // lanes currently leased
static size_t g_lanes_total = 0;   // lanes in existence (pooled + leased)
static int g_zero_copy = 0;            // DGX_ZERO_COPY=1: decode pinned packs in place over PCIe (off: DMA copies move the bytes faster)
constexpr size_t g_merge_multi_min = size_t(1) << 18;  // MergeSorted totals below this stay on the tree (fewer launches)
static int g_num_sms = 132;
constexpr size_t kPipeSmemMax = 220 * 1024;

// ---------------------------------------------------------------------------
// arenas
// ---------------------------------------------------------------------------
static cudaError_t pinned_alloc(void** p, size_t bytes);  // NUMA-aware cudaMallocHost (below)
static void numa_probe(int device);
// Device scratch: bump allocator, reset at the start of every public op (safe:
// later work on the same stream is ordered after earlier kernels).
struct DevArena {
    char* base = nullptr;
    size_t cap = 0, used = 0;
    std::vector<void*> retired;  // old chunks still referenced by queued work
    int alloc(size_t bytes, void** out) {
        bytes = (bytes + 255) & ~size_t(255);
        if (used + bytes > cap) {
            size_t ncap = std::max(cap * 2, used + bytes + (size_t(1) << 20));
            void* nb = nullptr;
            cudaError_t e = cudaMalloc(&nb, ncap);
            if (e != cudaSuccess) return fail(DGX_ERR_OOM, "cudaMalloc(%zu) failed: %s", ncap, cudaGetErrorString(e));
            if (base) retired.push_back(base);  // pointers handed out earlier in this op stay valid
            base = (char*)nb;
            cap = ncap;
            used = 0;
        }
        *out = base + used;
        used += bytes;
        return DGX_OK;
    }
    // Old chunks may still back pointers the current op hands to the host-side epilogue
    // (e.g. the D2H copy after a lane sync), so they are freed in two steps: a lane sync
    // makes them `freeable` (no queued work references them any more), the next op's
    // reset() actually frees them.
    std::vector<void*> freeable;
    void reset() {
        used = 0;
        for (void* p : freeable) cudaFree(p);
        freeable.clear();
    }
    void release_retired() {
        for (void* p : retired) freeable.push_back(p);
        retired.clear();
    }
    void destroy() {
        release_retired();
        for (void* p : freeable) cudaFree(p);
        freeable.clear();
        if (base) cudaFree(base);
        base = nullptr;
        cap = used = 0;
    }
};

// Pinned host staging for descriptor tables: async H2D copies read from it
// later, so it is only recycled at lane sync.
struct HostArena {
    struct Chunk { char* p; size_t cap, used; };
    std::vector<Chunk> chunks;
    int alloc(size_t bytes, void** out) {
        bytes = (bytes + 63) & ~size_t(63);
        if (chunks.empty() || chunks.back().used + bytes > chunks.back().cap) {
            size_t ncap = std::max(bytes, chunks.empty() ? (size_t(1) << 20) : chunks.back().cap * 2);
            void* p = nullptr;
            cudaError_t e = pinned_alloc(&p, ncap);
            if (e != cudaSuccess) return fail(DGX_ERR_OOM, "cudaMallocHost(%zu) failed: %s", ncap, cudaGetErrorString(e));
            chunks.push_back({(char*)p, ncap, 0});
        }
        Chunk& c = chunks.back();
        *out = c.p + c.used;
        c.used += bytes;
        return DGX_OK;
    }
    size_t used_bytes() const {
        size_t t = 0;
        for (const auto& c : chunks) t += c.used;
        return t;
    }
    void reset() {  // keep the largest (last) chunk
        while (chunks.size() > 1) {
            cudaFreeHost(chunks.front().p);
            chunks.erase(chunks.begin());
        }
        if (!chunks.empty()) chunks.back().used = 0;
    }
    void destroy() {
        for (auto& c : chunks) cudaFreeHost(c.p);
        chunks.clear();
    }
};

struct dgx_lane {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    DevArena ws;
    HostArena host;
    int* d_err = nullptr;   // device error flag (out_cap overflow)
    int* h_err = nullptr;   // pinned mirror
    uint64_t* h_word = nullptr;  // pinned scratch for lengths (8 words)
    uint64_t* h_head = nullptr;  // pinned landing zone for the head of a result (kSpecHead values)
    uint64_t launches = 0;
    uint64_t xm_overflows = 0;  // overflow-path chunks of the matrix merges this lane ran, as of its last sync
    uint64_t tail_queries = 0;  // filter queries with deferred lists this lane ran, as of its last sync
    // "resident lists" mode (dgx_lane_set_resident_inputs): the plan pre-pass of batch i+1 runs on a side stream while
    // the pipeline kernel of batch i is still running; its tables live in two alternating workspaces
    bool resident_inputs = false;
    cudaStream_t side = nullptr;
    DevArena fws[2];
    cudaEvent_t ev_plan[2] = {nullptr, nullptr}, ev_pipe[2] = {nullptr, nullptr};
    int fslot = 0;
    // Buffers the lane's own queued operations write (outputs of filter batches, merges, decodes since the last
    // dgx_lane_sync).  A batch that reads one of them is NOT planned ahead: its pre-pass is ordered behind the main
    // stream, so "decode -> intersect" or chained intersections on a resident-inputs lane stay correct.
    struct OutRange { const char* p; size_t bytes; };
    std::vector<OutRange> outs;
    bool outs_overflow = false;
    cudaEvent_t ev_prod = nullptr;
    void note_output(const void* p, size_t bytes) {
        if (!resident_inputs || !p || !bytes) return;
        for (OutRange& r : outs)
            if (r.p == (const char*)p) { r.bytes = std::max(r.bytes, bytes); return; }
        if (outs.size() >= 32) { outs_overflow = true; return; }
        outs.push_back({(const char*)p, bytes});
    }
    bool reads_own_output(const void* p) const {
        if (outs_overflow) return true;
        for (const OutRange& r : outs)
            if ((const char*)p >= r.p && (const char*)p < r.p + r.bytes) return true;
        return false;
    }
};
// Results up to this many values reach the host in the same round trip as their length.
constexpr size_t kSpecHead = 8192;

// Start of a device-level op on a lane: bind the device, recycle the workspace.  The pinned descriptor
// staging is only recycled at a lane sync (queued H2D copies read from it); a caller that queues thousands
// of ops without ever syncing would grow it without bound, so past a soft cap the op syncs the stream itself.
constexpr size_t kHostArenaSoftCap = size_t(16) << 20;
static int lane_begin_op(dgx_lane* l) {
    CK(cudaSetDevice(l->device));
    if (l->host.used_bytes() > kHostArenaSoftCap) {
        CK(cudaStreamSynchronize(l->stream));
        l->host.reset();
        l->ws.release_retired();
    }
    l->ws.reset();
    return DGX_OK;
}

// One call's scratch arrays carved from the lane's workspace by a WsLayout (ws_layout.hpp).  Declare the regions in
// section order; stage() places the copied section in the lane's pinned staging, where the caller fills the tables
// through the host pointers; commit() takes one arena allocation, uploads the copied section in one copy, sets the
// zeroed and ones sections with one memset each and writes every declared device pointer.
class WsCarve {
  public:
    explicit WsCarve(dgx_lane* l) : l_(l) {}
    template <class D, class H>
    void copied(D** d, H** h, size_t n) {
        static_assert(sizeof(D) == sizeof(H) && alignof(D) == alignof(H), "device and host views of one table");
        if (h_) L_.ok = false;  // the staged section cannot grow
        const size_t off = L_.add<H>(WsLayout::kCopied, n);
        put(d, off, false);
        put(h, off, true);
    }
    template <class T> void zeroed(T** d, size_t n) { put(d, L_.add<T>(WsLayout::kZeroed, n), false); }
    template <class T> void ones(T** d, size_t n) { put(d, L_.add<T>(WsLayout::kOnes, n), false); }
    template <class T> void plain(T** d, size_t n) { put(d, L_.add<T>(WsLayout::kPlain, n), false); }

    int stage() {
        const size_t nc = L_.end(WsLayout::kCopied);
        if (int rc = l_->host.alloc(nc, (void**)&h_)) return rc;
        bind(h_, true);
        return DGX_OK;
    }
    int commit() {
        const size_t nc = L_.end(WsLayout::kCopied);
        if (!L_.ok || nslots_ > kMaxSlots || (nc && !h_))
            return fail(DGX_ERR_CUDA, "workspace layout: a region out of section order, or its table not staged");
        char* d;
        if (int rc = l_->ws.alloc(L_.bytes, (void**)&d)) return rc;
        if (nc) {
            CK(cudaMemcpyAsync(d, h_, nc, cudaMemcpyHostToDevice, l_->stream));
            g_stats.h2d += nc;
        }
        for (int s : {int(WsLayout::kZeroed), int(WsLayout::kOnes)})
            if (L_.end(s) > L_.begin(s))
                CK(cudaMemsetAsync(d + L_.begin(s), s == WsLayout::kOnes ? 0xff : 0, L_.end(s) - L_.begin(s), l_->stream));
        bind(d, false);
        return DGX_OK;
    }

  private:
    static constexpr int kMaxSlots = 48;
    struct Slot { void* p; void (*set)(void*, char*); size_t off; bool host; };
    template <class T>
    void put(T** p, size_t off, bool host) {
        if (nslots_ < kMaxSlots) slots_[nslots_] = {p, [](void* s, char* b) { *(T**)s = (T*)b; }, off, host};
        ++nslots_;
    }
    void bind(char* base, bool host) {
        for (int i = 0; i < std::min(nslots_, kMaxSlots); ++i)
            if (slots_[i].host == host) slots_[i].set(slots_[i].p, base + slots_[i].off);
    }
    dgx_lane* l_;
    WsLayout L_;
    char* h_ = nullptr;
    Slot slots_[kMaxSlots];
    int nslots_ = 0;
};

// ---------------------------------------------------------------------------
// lifecycle
// ---------------------------------------------------------------------------
extern "C" int dgx_init(int device) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_device >= 0) return DGX_OK;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(DGX_ERR_NODEV, "no CUDA device: %s", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    if (device < 0) {
        if (cudaGetDevice(&device) != cudaSuccess) device = 0;
    }
    if (device >= n) return fail(DGX_ERR_ARG, "device %d out of range (%d devices)", device, n);
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    // the library carries sm_90a code only (no PTX), which loads on compute capability 9.0 and nothing else
    if (prop.major != 9 || prop.minor != 0)
        return fail(DGX_ERR_NODEV, "libdgx is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
    CK(cudaFuncSetAttribute(decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)(sizeof(DWarpSmem) * D_WARPS)));
    CK(cudaFuncSetAttribute(decode_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)(sizeof(DWarpSmem) * D_WARPS)));
    CK(cudaFuncSetAttribute(icw_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)(sizeof(DWarpSmem) * D_WARPS)));
    CK(cudaFuncSetAttribute(filter_pipe_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPipeSmemMax));
    CK(cudaFuncSetAttribute(filter_pipe_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPipeSmemMax));
    g_num_sms = prop.multiProcessorCount;
    numa_probe(device);
    CK(cudaFuncSetAttribute(mmerge3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T_SMEM));
    if (const char* s = getenv("DGX_ZERO_COPY")) g_zero_copy = atoi(s) != 0;
    g_device = device;
    return DGX_OK;
}

extern "C" void dgx_shutdown(void) {
    dgx_cache_clear();
    std::unique_lock<std::mutex> lk(g_mu);
    g_pool_cv.wait(lk, [] { return g_lanes_out == 0; });  // calls in flight keep their lanes until they return
    for (dgx_lane* l : g_pool) dgx_lane_destroy(l);
    g_pool.clear();
    g_lanes_total = 0;
    g_device = -1;
}

extern "C" int dgx_describe(char* buf, size_t n) {
    int rc = dgx_init(-1);
    if (rc != DGX_OK) return rc;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, g_device));
    snprintf(buf, n, "libdgx sm_90a | device %d: %s, %d SMs, %.1f GB | filter tiles %d / %d, merge tile %d",
             g_device, prop.name, prop.multiProcessorCount, prop.totalGlobalMem / 1e9, p_tile_size(2), p_tile_size(4), M_T);
    return DGX_OK;
}

// Pinned host memory is placed on the NUMA node the GPU hangs off: a DMA from the far socket runs at
// about half the PCIe rate.  While the pages are allocated the calling thread is moved to the GPU's
// node (first touch) and, where the container allows it, the memory policy prefers that node; both
// are restored afterwards and every step is best effort (DGX_NUMA=0 turns it off).
static int g_numa_node = -2;  // -2 unknown, -1 none
static cpu_set_t g_numa_cpus;
static void numa_probe(int device) {
    g_numa_node = -1;
    if (const char* s = getenv("DGX_NUMA")) if (atoi(s) == 0) return;
    char bus[32] = {0}, path[128];
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) return;
    for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    int node = -1;
    if (f) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
    if (node < 0) return;
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return;
    CPU_ZERO(&g_numa_cpus);
    int a, b, n = 0;
    while (fscanf(f, "%d", &a) == 1) {
        b = a;
        int c = fgetc(f);
        if (c == '-') { if (fscanf(f, "%d", &b) != 1) b = a; c = fgetc(f); }
        for (int i = a; i <= b && i < CPU_SETSIZE; ++i) { CPU_SET(i, &g_numa_cpus); ++n; }
        if (c != ',') break;
    }
    fclose(f);
    if (n) g_numa_node = node;
}
static cudaError_t pinned_alloc(void** p, size_t bytes) {
    cpu_set_t old;
    bool moved = false, policy = false;
    if (g_numa_node >= 0) {
        if (sched_getaffinity(0, sizeof(old), &old) == 0 && sched_setaffinity(0, sizeof(g_numa_cpus), &g_numa_cpus) == 0) moved = true;
        unsigned long mask[16] = {0};
        if (g_numa_node < 1024) {
            mask[g_numa_node / (8 * sizeof(unsigned long))] |= 1ul << (g_numa_node % (8 * sizeof(unsigned long)));
            policy = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, 1024ul) == 0;
        }
    }
    const cudaError_t e = cudaMallocHost(p, bytes ? bytes : 1);
    if (policy) syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0ul);
    if (moved) sched_setaffinity(0, sizeof(old), &old);
    return e;
}

extern "C" void* dgx_host_alloc(size_t bytes) {
    if (dgx_init(-1) != DGX_OK) return nullptr;
    void* p = nullptr;
    if (pinned_alloc(&p, bytes) != cudaSuccess) return nullptr;
    return p;
}
extern "C" void dgx_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

extern "C" void dgx_get_stats(dgx_stats* out) {
    out->calls = g_stats.calls;
    out->uids_in = g_stats.uids_in;
    out->uids_out = g_stats.uids_out;
    out->h2d_bytes = g_stats.h2d;
    out->d2h_bytes = g_stats.d2h;
    out->kernel_launches = g_stats.launches;
}

extern "C" dgx_lane* dgx_lane_create(int device, void* stream) {
    if (dgx_init(device) != DGX_OK) return nullptr;
    if (device < 0) device = g_device;
    // One device per process (one alpha process per GPU): kernel attributes, the SM count and the
    // host-pointer entry points are bound to the device dgx_init chose.
    if (device != g_device) {
        fail(DGX_ERR_ARG, "libdgx is bound to device %d in this process; lane requested on device %d", g_device, device);
        return nullptr;
    }
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    dgx_lane* l = new dgx_lane();
    l->device = device;
    if (stream) {
        l->stream = (cudaStream_t)stream;
    } else {
        if (cudaStreamCreateWithFlags(&l->stream, cudaStreamNonBlocking) != cudaSuccess) { delete l; return nullptr; }
        l->own_stream = true;
    }
    if (cudaMalloc(&l->d_err, 256) != cudaSuccess ||
        pinned_alloc((void**)&l->h_err, 4096 + kSpecHead * sizeof(uint64_t)) != cudaSuccess) {
        fail(DGX_ERR_OOM, "lane allocation failed");
        delete l;
        return nullptr;
    }
    l->h_word = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(l->h_err) + 64);
    l->h_head = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(l->h_err) + 4096);
    *l->h_err = 0;
    cudaMemsetAsync(l->d_err, 0, 256, l->stream);
    return l;
}

extern "C" void dgx_lane_destroy(dgx_lane* l) {
    if (!l) return;
    cudaSetDevice(l->device);
    cudaStreamSynchronize(l->stream);
    l->ws.destroy();
    l->host.destroy();
    if (l->d_err) cudaFree(l->d_err);
    if (l->h_err) cudaFreeHost(l->h_err);
    if (l->side) { cudaStreamSynchronize(l->side); cudaStreamDestroy(l->side); }
    for (int i = 0; i < 2; ++i) {
        l->fws[i].destroy();
        if (l->ev_plan[i]) cudaEventDestroy(l->ev_plan[i]);
        if (l->ev_pipe[i]) cudaEventDestroy(l->ev_pipe[i]);
        if (i == 0 && l->ev_prod) cudaEventDestroy(l->ev_prod);
    }
    if (l->own_stream) cudaStreamDestroy(l->stream);
    delete l;
}

extern "C" void* dgx_lane_stream(dgx_lane* l) { return l ? (void*)l->stream : nullptr; }

extern "C" int dgx_lane_set_resident_inputs(dgx_lane* l, int on) {
    if (!l) return fail(DGX_ERR_ARG, "null lane");
    CK(cudaSetDevice(l->device));
    if (on && !l->side) {
        CK(cudaStreamCreateWithFlags(&l->side, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            CK(cudaEventCreateWithFlags(&l->ev_plan[i], cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&l->ev_pipe[i], cudaEventDisableTiming));
        }
        CK(cudaEventCreateWithFlags(&l->ev_prod, cudaEventDisableTiming));
    }
    if (!on && l->side) CK(cudaStreamSynchronize(l->side));
    l->resident_inputs = on != 0;
    return DGX_OK;
}
extern "C" uint64_t dgx_lane_launches(const dgx_lane* l) { return l ? l->launches : 0; }

extern "C" int dgx_lane_sync(dgx_lane* l) {
    if (!l) return fail(DGX_ERR_ARG, "null lane");
    CK(cudaSetDevice(l->device));
    static_assert(kLaneTailWord == kLaneOverflowWord + 1, "the lane's counter words are read back in one copy");
    CK(cudaMemcpyAsync(l->h_err, l->d_err, (kLaneTailWord + 1) * sizeof(u32), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    l->host.reset();
    l->ws.release_retired();
    l->outs.clear();
    l->outs_overflow = false;
    if (const u32 ovf = reinterpret_cast<const u32*>(l->h_err)[kLaneOverflowWord]) {
        l->xm_overflows += ovf;
        g_xm_overflows += ovf;
        CK(cudaMemsetAsync(reinterpret_cast<u32*>(l->d_err) + kLaneOverflowWord, 0, sizeof(u32), l->stream));
    }
    if (const u32 tq = reinterpret_cast<const u32*>(l->h_err)[kLaneTailWord]) {
        l->tail_queries += tq;
        g_tail_queries += tq;
        CK(cudaMemsetAsync(reinterpret_cast<u32*>(l->d_err) + kLaneTailWord, 0, sizeof(u32), l->stream));
    }
    if (const int flag = *l->h_err) {
        *l->h_err = 0;
        CK(cudaMemsetAsync(l->d_err, 0, sizeof(int), l->stream));
        if (flag & kLaneErrOrder) return fail(DGX_ERR_ARG, "a row of the uid matrix is not strictly ascending");
        if (flag & kLaneErrVarint) return fail(DGX_ERR_ARG, "a uid_bytes row is not a sequence of valid uvarints");
        if (flag & kLaneErrGroupBy)
            return fail(DGX_ERR_ARG, "a groupby input is malformed (src, a row, a parent row or dest not strictly "
                                     "ascending, offsets not starting at 0, decreasing or past their arrays, a row "
                                     "value missing from dest, or 2^32 restricted edges or more)");
        if (flag & kLaneErrRecurse)
            return fail(DGX_ERR_ARG, "a recurse step's input is malformed (src, a row or dest not strictly ascending, "
                                     "or offsets not starting at 0, decreasing or past v_cap)");
        if (flag & kLaneErrCascade)
            return fail(DGX_ERR_ARG, "a cascade input is malformed (a dest or an unordered row not strictly ascending, "
                                     "or row offsets not starting at 0, decreasing or past v_cap)");
        if (flag & kLaneErrPath)
            return fail(DGX_ERR_ARG, "a shortest-path level's input is malformed (src, a row or a dest not strictly "
                                     "ascending, offsets not starting at 0, decreasing or past their caps, or a source "
                                     "with a kept edge not discovered at the previous level)");
        if (flag & kLaneErrVar)
            return fail(DGX_ERR_ARG, "a value-variable input is malformed (map keys, src or dest not strictly ascending, "
                                     "offsets not starting at 0, decreasing or past v_cap, or a row value missing from "
                                     "its level's dest)");
        if (flag & kLaneErrMath)
            return fail(DGX_ERR_ARG, "a math() input is refused (leaf keys or range not strictly ascending, an unknown "
                                     "tag, a count word past its room, key 0 among other keys, or a result Go "
                                     "returns as an error or computes in map-iteration order)");
        if (flag & kLaneErrSgFilter)
            return fail(DGX_ERR_ARG, "an @filter input is malformed (d0, a row or a LIST leaf not strictly ascending, "
                                     "a COUNT leaf's offsets or the row offsets decreasing, row offsets not starting "
                                     "at 0 or past v_cap, or a length word past its room)");
        if (flag & kLaneErrVarOrder)
            return fail(DGX_ERR_ARG, "an order-by-variable input is refused (dest, map keys or a row not strictly "
                                     "ascending, row offsets not starting at 0, decreasing or past v_cap, a length word "
                                     "past its room, an unknown entry tag, or a row whose first mapped entry is a bool, "
                                     "which Go refuses as not sortable)");
        if (flag & kLaneErrMatch)
            return fail(DGX_ERR_ARG, "a match() input is malformed (candidates or column uids not strictly ascending, "
                                     "column offsets not starting at 0, decreasing or not ending at nvals / nbytes, or "
                                     "a length word past its room; regexp()'s value test shares these checks)");
        if (flag & kLaneErrCompare)
            return fail(DGX_ERR_ARG, "a compare function's input is refused (candidates or column uids not strictly "
                                     "ascending, column or row offsets malformed, a length word past its room, or a "
                                     "candidate's value whose conversion failed)");
        if (flag & kLaneErrPredOrder)
            return fail(DGX_ERR_ARG, "an order-by-predicate input is refused (dest, a row or column uids not strictly "
                                     "ascending, row or column offsets malformed, a length word past its room, a "
                                     "row uid owning several values, which Go refuses as a list predicate, or a "
                                     "datetime value's nanoseconds of 10^9 or more)");
        if (flag & kLaneErrMut)
            return fail(DGX_ERR_ARG, "a mutable layer is malformed (entries not strictly ascending, uid 0 or unknown "
                                     "flags) or a probe / iterate / unfiltered row's pack starts at uid 0");
        return fail(DGX_ERR_CAP, "result does not fit out_cap");
    }
    return DGX_OK;
}

extern "C" void* dgx_dev_alloc(size_t bytes) {
    if (dgx_init(-1) != DGX_OK) return nullptr;
    void* p = nullptr;
    if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) { fail(DGX_ERR_OOM, "cudaMalloc(%zu) failed", bytes); return nullptr; }
    return p;
}
extern "C" void dgx_dev_free(void* p) {
    if (p) cudaFree(p);
}
extern "C" int dgx_memcpy_h2d(dgx_lane* l, void* d, const void* h, size_t bytes) {
    if (!l) return fail(DGX_ERR_ARG, "null lane");
    CK(cudaSetDevice(l->device));
    if (bytes) CK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += bytes;
    return DGX_OK;
}
extern "C" int dgx_memcpy_d2h(dgx_lane* l, void* h, const void* d, size_t bytes) {
    if (!l) return fail(DGX_ERR_ARG, "null lane");
    CK(cudaSetDevice(l->device));
    if (bytes) CK(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, l->stream));
    g_stats.d2h += bytes;
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// filter (intersect / k-way intersect / difference), device level
// ---------------------------------------------------------------------------
struct ListDesc {
    const uint64_t* ptr;
    size_t len;
    const uint64_t* dyn_len;
};

// Queries q own lists [k_off[q], k_off[q+1]).  Results -> d_out / d_out_off.
static int filter_batch_impl(dgx_lane* l, int op, const ListDesc* lists, const size_t* k_off, size_t nq,
                             uint64_t* d_out, size_t out_cap, uint64_t* d_out_off) {
    if (nq == 0) {
        CK(cudaMemsetAsync(d_out_off, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    const size_t nlists = k_off[nq] - k_off[0];
    void *h_raw, *d_raw;
    const size_t tasks_b = nq * sizeof(FTask), lists_b = (nlists + 1) * sizeof(FList);
    int rc = l->host.alloc(tasks_b + lists_b, &h_raw);
    if (rc) return rc;
    FTask* ht = (FTask*)h_raw;
    FList* hl = (FList*)((char*)h_raw + tasks_b);
    uint64_t ntiles = 0, uids_in = 0, mid_cap = 0;
    size_t li = 0, kmax = 1;
    bool sample_any = false;
    for (size_t q = 0; q < nq; ++q) kmax = std::max(kmax, k_off[q + 1] - k_off[q]);
    // 1- and 2-list batches: 1024-value tiles (per-tile overheads over twice the values); wider queries: 512 (filter_pipe.cuh)
    const int pipe_va = kmax <= 2 ? 4 : 2;
    const uint64_t tile_sz = (uint64_t)p_tile_size(pipe_va);
    std::vector<size_t> order;
    for (size_t q = 0; q < nq; ++q) {
        const size_t k0 = k_off[q], k1 = k_off[q + 1];
        const size_t k = k1 - k0;
        if (k == 0) return fail(DGX_ERR_ARG, "query %zu has no lists", q);
        if (op == DGX_OP_DIFFERENCE && k != 2) return fail(DGX_ERR_ARG, "difference takes exactly two lists");
        order.resize(k);
        std::iota(order.begin(), order.end(), k0);
        if (op == DGX_OP_INTERSECT)  // drive from the shortest list (algo/uidlist.go:309-311)
            std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) { return lists[x].len < lists[y].len; });
        ht[q].tile_base = ntiles;
        ht[q].list_first = (u32)li;
        ht[q].k = (u32)k;
        for (size_t i = 0; i < k; ++i) {
            const ListDesc& L = lists[order[i]];
            hl[li].ptr = (const u64*)L.ptr;
            hl[li].len = L.len;
            hl[li].dyn_len = (const u64*)L.dyn_len;
            uids_in += L.len;
            ++li;
        }
        const uint64_t lenA = lists[order[0]].len;
        ntiles += std::max<uint64_t>(1, (lenA + tile_sz - 1) / tile_sz);
        mid_cap += lenA;
        sample_any |= k >= 3 && lenA >= P_SAMPLE_MIN_A;
    }
    if (ntiles > 0x7fffffffull) return fail(DGX_ERR_ARG, "batch too large (%llu tiles)", (unsigned long long)ntiles);
    const bool ahead = l->resident_inputs && l->side;
    // Intersections of 3+ lists on a resident-inputs lane, where the pre-pass runs under the previous batch's
    // pipeline, are sampled and may defer their sparse tail to filter_tail_kernel (filter_pipe.cuh).  Elsewhere
    // the sample would sit on the call's critical path, and driving lists under P_SAMPLE_MIN_A values (an upper
    // bound here; the sample checks the exact length) are not worth sampling.
    const bool deep = op == DGX_OP_INTERSECT && ahead && sample_any;
    // zeroed per batch: pipeline status words | 64 B (pipeline ticket, deferral word, tail ticket) | deep batches:
    // tail status words, the sample's hit words (P_SAMPLES per query) and its per-query CTA counts
    const uint64_t tail_chunks = mid_cap / P_TAIL_NT + 1;
    if (deep && tail_chunks > 0xffffffffull) return fail(DGX_ERR_ARG, "batch too large (%llu values)", (unsigned long long)mid_cap);
    const size_t sample_b = nq * (P_SAMPLES + 1) * sizeof(u32);
    const size_t status_b = ntiles * sizeof(u64) + 64 + (deep ? tail_chunks * sizeof(u64) + sample_b : 0);
    // Where the batch's tables live and which stream prepares them.  Normally: the lane's workspace and stream.
    // Resident-inputs lanes: one of two alternating workspaces and the side stream -- descriptor copies, status
    // reset and the plan pre-pass of THIS batch then run while the pipeline kernel of the PREVIOUS batch is still
    // busy (the lists are immutable, so the pre-pass depends on nothing the main stream has queued).
    const int slot = l->fslot;
    DevArena* ar = &l->ws;
    cudaStream_t pre = l->stream;
    if (ahead) {
        l->fslot ^= 1;
        ar = &l->fws[slot];
        pre = l->side;
        CK(cudaStreamWaitEvent(l->side, l->ev_pipe[slot], 0));  // the pipeline that last read this workspace is done
        bool dep = false;  // a list this lane's own queued work produces: plan it behind that work, not ahead
        for (size_t i = k_off[0]; i < k_off[nq] && !dep; ++i)
            dep = l->reads_own_output(lists[i].ptr) || (lists[i].dyn_len && l->reads_own_output(lists[i].dyn_len));
        if (dep) {
            CK(cudaEventRecord(l->ev_prod, l->stream));
            CK(cudaStreamWaitEvent(l->side, l->ev_prod, 0));
        }
        ar->reset();
    }
    rc = ar->alloc(tasks_b + lists_b + status_b, &d_raw);
    if (rc) return rc;
    CK(cudaMemcpyAsync(d_raw, h_raw, tasks_b + lists_b, cudaMemcpyHostToDevice, pre));
    char* d_status = (char*)d_raw + tasks_b + lists_b;
    CK(cudaMemsetAsync(d_status, 0, status_b, pre));
    FParams P;
    P.tasks = (const FTask*)d_raw;
    P.lists = (const FList*)((char*)d_raw + tasks_b);
    P.ntasks = (u32)nq;
    P.ntiles = (u32)ntiles;
    P.op = op;
    P.out = (u64*)d_out;
    P.out_cap = out_cap;
    P.out_off = (u64*)d_out_off;
    P.status = (u64*)d_status;
    P.ticket = (u32*)(d_status + ntiles * sizeof(u64));
    P.err = l->d_err;
    u32* d_defer = P.ticket + 1;
    u32* d_tail_ticket = P.ticket + 2;
    u64* d_tail_status = (u64*)(d_status + ntiles * sizeof(u64) + 64);
    u32* d_hits = (u32*)(d_tail_status + (deep ? tail_chunks : 0));
    u32* d_done = d_hits + nq * P_SAMPLES;
    // ---- stream depth per query (deep batches): k_eff words, the intermediate and its offsets --------
    void *d_keff = nullptr, *d_mid = nullptr, *d_mid_off = nullptr;
    if (deep) {
        rc = ar->alloc(nq * sizeof(u32), &d_keff);
        if (rc) return rc;
        rc = ar->alloc(std::max<uint64_t>(mid_cap, 1) * sizeof(u64), &d_mid);
        if (rc) return rc;
        rc = ar->alloc((nq + 1) * sizeof(u64), &d_mid_off);
        if (rc) return rc;
        const dim3 sgrid((unsigned)nq, (unsigned)std::min<size_t>(kmax - 2, P_SAMPLE_LISTS));
        filter_sample_kernel<<<sgrid, P_SAMPLES, 0, pre>>>(P.tasks, P.lists, d_hits, d_done, (u32*)d_keff, d_defer);
        CK(cudaGetLastError());
        l->launches += 1;
        g_stats.launches += 1;
    }
    // ---- plan pre-pass + persistent TMA pipeline (filter_pipe_kernel) ----------------
    void* hp_raw;
    rc = l->host.alloc(nq * sizeof(u64), &hp_raw);
    if (rc) return rc;
    u64* h_pb = (u64*)hp_raw;
    u64 npairs = 0;
    for (size_t q = 0; q < nq; ++q) {
        h_pb[q] = npairs;
        const u64 nt = (q + 1 < nq ? ht[q + 1].tile_base : ntiles) - ht[q].tile_base;
        npairs += nt * (u64)(ht[q].k - 1);
    }
    void *d_pb, *d_plan, *d_tiles;
    rc = ar->alloc(nq * sizeof(u64), &d_pb);
    if (rc) return rc;
    rc = ar->alloc(ntiles * sizeof(PTileEntry), &d_tiles);
    if (rc) return rc;
    rc = ar->alloc((npairs + 1) * sizeof(PPlanEntry), &d_plan);
    if (rc) return rc;
    CK(cudaMemcpyAsync(d_pb, h_pb, nq * sizeof(u64), cudaMemcpyHostToDevice, pre));
    filter_tiles_kernel<<<(unsigned)((ntiles + 255) / 256), 256, 0, pre>>>(P.tasks, P.lists, (const u64*)d_pb, P.ntasks,
                                                                           P.ntiles, (PTileEntry*)d_tiles, (u32)tile_sz,
                                                                           (const u32*)d_keff);
    CK(cudaGetLastError());
    l->launches += 1;
    g_stats.launches += 1;
    if (npairs) {  // a batch of one-list queries has no slices to bound
        const u64 blocks = (npairs + 255) / 256;
        if (blocks > 0x7fffffffull) return fail(DGX_ERR_ARG, "batch too large");
        filter_plan_kernel<<<(unsigned)blocks, 256, 0, pre>>>(P.tasks, P.lists, (const u64*)d_pb, P.ntasks, npairs,
                                                              (PPlanEntry*)d_plan, (u32)tile_sz, (const u32*)d_keff);
        CK(cudaGetLastError());
        l->launches += 1;
        g_stats.launches += 1;
    }
    PParams PP;
    PP.f = P;
    PP.plan_base = (const u64*)d_pb;
    PP.plan = (const PPlanEntry*)d_plan;
    PP.tiles = (const PTileEntry*)d_tiles;
    PP.defer = deep ? d_defer : nullptr;
    PP.mid = (u64*)d_mid;
    PP.mid_off = (u64*)d_mid_off;
    PP.mid_cap = mid_cap;
    // wide queries: one tile per ticket keeps the look-back order tight; 2-list batches have tiny tiles and
    // amortise the metadata chain over two
    PP.grp = kmax >= 4 ? 1u : 2u;
    const size_t nl = std::min<size_t>(std::max<size_t>(kmax - 1, 1), P_MAXL);
    const size_t TA = (size_t)tile_sz;
    // staged slices: ~1.125 tile-widths per filter list; a 2-list batch stages up to 2.25 tile-widths of its one
    // filter list (size ratios beyond that probe the list in HBM, the reference's own Jump / Bin regimes)
    size_t cap = (TA + TA / 8) * nl * (kmax <= 2 ? 2 : 1);
    cap = std::min<size_t>(std::max<size_t>(cap, TA + TA / 8), 9216) & ~size_t(1);
    PP.slice_cap = (u32)cap;
    const size_t smem = ((sizeof(PShared) + 127) & ~size_t(127)) + (1 + P_OS) * TA * sizeof(u64) +
                        P_ST * ((TA + 2) + cap) * sizeof(u64);
    if (smem > kPipeSmemMax) return fail(DGX_ERR_ARG, "pipeline stage too large");
    auto kern = pipe_va == 4 ? filter_pipe_kernel<4> : filter_pipe_kernel<2>;
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, P_NT, smem));
    if (per_sm < 1) return fail(DGX_ERR_CUDA, "filter_pipe_kernel does not fit on an SM");
    PP.nctas = (u32)std::min<u64>((u64)per_sm * (u64)g_num_sms, ntiles);
    if (ahead) {
        CK(cudaEventRecord(l->ev_plan[slot], l->side));
        CK(cudaStreamWaitEvent(l->stream, l->ev_plan[slot], 0));
    }
    kern<<<PP.nctas, P_NT, smem, l->stream>>>(PP);
    CK(cudaGetLastError());
    l->launches += 1;
    g_stats.launches += 1;
    if (deep) {  // exits at once unless the sample deferred some query
        PTailParams T;
        T.tasks = P.tasks;
        T.lists = P.lists;
        T.ntasks = P.ntasks;
        T.keff = (const u32*)d_keff;
        T.defer = d_defer;
        T.mid = (const u64*)d_mid;
        T.mid_off = (const u64*)d_mid_off;
        T.out = P.out;
        T.out_cap = P.out_cap;
        T.out_off = P.out_off;
        T.status = d_tail_status;
        T.ticket = d_tail_ticket;
        T.err = l->d_err;
        T.tail_queries = (u32*)l->d_err + kLaneTailWord;
        const u64 ctas = std::min<u64>((u64)g_num_sms * (2048 / P_TAIL_NT), tail_chunks);
        filter_tail_kernel<<<(unsigned)ctas, P_TAIL_NT, 0, l->stream>>>(T);
        CK(cudaGetLastError());
        l->launches += 1;
        g_stats.launches += 1;
    }
    // the tail reads this workspace too: the pre-pass that reuses it waits for both
    if (ahead) CK(cudaEventRecord(l->ev_pipe[slot], l->stream));
    g_stats.uids_in += uids_in;
    return DGX_OK;
}

extern "C" int dgx_dev_filter_batch(dgx_lane* l, int op, const uint64_t* const* d_lists, const size_t* lens,
                                    const size_t* k_off, size_t nq, uint64_t* d_out, size_t out_cap,
                                    uint64_t* d_out_off) {
    if (!l || (op != DGX_OP_INTERSECT && op != DGX_OP_DIFFERENCE)) return fail(DGX_ERR_ARG, "bad lane/op");
    if (int rc = lane_begin_op(l)) return rc;
    const size_t nlists = nq ? k_off[nq] : 0;
    std::vector<ListDesc> ld(nlists);
    for (size_t i = 0; i < nlists; ++i) ld[i] = {d_lists[i], lens[i], nullptr};
    g_stats.calls += 1;
    const int rc = filter_batch_impl(l, op, ld.data(), k_off, nq, d_out, out_cap, d_out_off);
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_out_off, (nq + 1) * sizeof(uint64_t));
    return rc;
}

// ---------------------------------------------------------------------------
// MergeSorted, device level: tree of batched 2-way unions
// ---------------------------------------------------------------------------
static int merge_tree_impl(dgx_lane* l, std::vector<MRef> cur, std::vector<uint64_t> ub, uint64_t total,
                           uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);
static int merge_multi_impl(dgx_lane* l, const std::vector<MRef>& runs, const std::vector<uint64_t>& ub, uint64_t total,
                            uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);
static int merge_runs_impl(dgx_lane* l, const std::vector<MRef>& cur, const std::vector<uint64_t>& ub, uint64_t total,
                           uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);

static int merge_sorted_impl(dgx_lane* l, const ListDesc* lists, size_t k, uint64_t* d_out, size_t out_cap,
                             uint64_t* d_out_len) {
    // nil / empty lists are skipped (algo/uidlist.go:400-403)
    std::vector<MRef> cur;
    std::vector<uint64_t> ub;
    uint64_t total = 0;
    for (size_t i = 0; i < k; ++i) {
        if (lists[i].ptr == nullptr || lists[i].len == 0) continue;
        cur.push_back(MRef{(const u64*)lists[i].ptr, nullptr, (u64)lists[i].len});
        ub.push_back(lists[i].len);
        total += lists[i].len;
    }
    g_stats.uids_in += total;
    if (cur.empty()) {
        CK(cudaMemsetAsync(d_out_len, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (out_cap < total) return fail(DGX_ERR_CAP, "MergeSorted needs out_cap >= sum(lens) = %llu", (unsigned long long)total);
    return merge_runs_impl(l, cur, ub, total, d_out, out_cap, d_out_len);
}

// Dispatch over the number of runs: the single-pass multiway merge for 3..64 large runs, groups of <= 64 runs merged
// multiway into intermediate runs (whose lengths stay on the device: MRef::off) and merged again for more -- two passes
// over HBM up to 4096 runs instead of ceil(log2 k) -- and the pairwise tree for everything small.
static int merge_runs_impl(dgx_lane* l, const std::vector<MRef>& cur, const std::vector<uint64_t>& ub, uint64_t total,
                           uint64_t* d_out, size_t out_cap, uint64_t* d_out_len) {
    const size_t k = cur.size();
    if (k >= 3 && k <= (size_t)MM_K && total >= g_merge_multi_min)
        return merge_multi_impl(l, cur, ub, total, d_out, out_cap, d_out_len);
    const size_t ngroups = (k + MM_K - 1) / MM_K;
    // a multiway call is a dozen launches: grouping pays only when every group is a few times the multiway minimum
    if (k <= (size_t)MM_K || total / ngroups < 4 * g_merge_multi_min)
        return merge_tree_impl(l, cur, ub, total, d_out, out_cap, d_out_len);
    const size_t gsz = (k + ngroups - 1) / ngroups;
    void *d_tmp, *d_pairs;
    int rc = l->ws.alloc(total * sizeof(u64), &d_tmp);
    if (rc) return rc;
    rc = l->ws.alloc(2 * ngroups * sizeof(u64), &d_pairs);
    if (rc) return rc;
    CK(cudaMemsetAsync(d_pairs, 0, 2 * ngroups * sizeof(u64), l->stream));
    std::vector<MRef> next;
    std::vector<uint64_t> nub;
    uint64_t goff = 0;
    for (size_t g = 0; g < ngroups; ++g) {
        const size_t b = g * gsz, e = std::min(k, b + gsz);
        if (b >= e) break;
        std::vector<MRef> part(cur.begin() + b, cur.begin() + e);
        std::vector<uint64_t> pub(ub.begin() + b, ub.begin() + e);
        uint64_t tot = 0;
        for (uint64_t v : pub) tot += v;
        u64* dst = (u64*)d_tmp + goff;
        u64* pair = (u64*)d_pairs + 2 * g;  // {0, length of the group's merged run}
        rc = merge_runs_impl(l, part, pub, tot, (uint64_t*)dst, tot, (uint64_t*)(pair + 1));
        if (rc) return rc;
        next.push_back(MRef{dst, pair, (u64)tot});
        nub.push_back(tot);
        goff += tot;
    }
    return merge_runs_impl(l, next, nub, total, d_out, out_cap, d_out_len);
}

// Pairwise merge tree: ceil(log2 k) passes of merge_kernel.
static int merge_tree_impl(dgx_lane* l, std::vector<MRef> cur, std::vector<uint64_t> ub, uint64_t total,
                           uint64_t* d_out, size_t out_cap, uint64_t* d_out_len) {
    // number of levels; a single list still takes one pass (in-list de-duplication)
    int levels = 0;
    for (size_t n = cur.size(); n > 1; n = (n + 1) / 2) ++levels;
    if (levels == 0) levels = 1;
    void* d_tmp = nullptr;
    int rc;
    if (levels > 1) {
        rc = l->ws.alloc(total * sizeof(u64), &d_tmp);
        if (rc) return rc;
    }
    // plan all levels on the host
    struct Level { std::vector<MTask> tasks; uint64_t ntiles; u64* out; size_t off_index; };
    std::vector<Level> plan(levels);
    size_t off_words = 0, task_count = 0;
    uint64_t tiles_total = 0;
    for (int lv = 0; lv < levels; ++lv) {
        Level& L = plan[lv];
        L.out = ((levels - 1 - lv) % 2 == 0) ? (u64*)d_out : (u64*)d_tmp;
        const size_t n = cur.size();
        const size_t nt = (n + 1) / 2;
        L.tasks.resize(nt);
        L.ntiles = 0;
        L.off_index = off_words;
        std::vector<uint64_t> nub(nt);
        for (size_t t = 0; t < nt; ++t) {
            MTask& T = L.tasks[t];
            T.tile_base = L.ntiles;
            T.a = cur[2 * t];
            uint64_t u = ub[2 * t];
            if (2 * t + 1 < n) { T.b = cur[2 * t + 1]; u += ub[2 * t + 1]; }
            else T.b = MRef{nullptr, nullptr, 0};
            nub[t] = u;
            L.ntiles += std::max<uint64_t>(1, (u + M_T - 1) / M_T);
        }
        if (L.ntiles > 0x7fffffffull) return fail(DGX_ERR_ARG, "merge too large");
        off_words += nt + 1;
        task_count += nt;
        tiles_total += L.ntiles;
        // next level's inputs are slices of this level's compact output (offsets patched below)
        cur.assign(nt, MRef{L.out, nullptr, 0});
        ub = nub;
        for (size_t t = 0; t < nt; ++t) { cur[t].len = nub[t]; cur[t].off = (const u64*)(uintptr_t)(L.off_index + t + 1); }
    }
    // device layout: [off words][tasks][status + tickets]
    const size_t off_b = off_words * sizeof(u64);
    const size_t tasks_b = task_count * sizeof(MTask);
    const size_t status_b = (tiles_total + 2 * levels) * sizeof(u64);
    void *d_raw, *h_raw;
    rc = l->ws.alloc(off_b + tasks_b + status_b, &d_raw);
    if (rc) return rc;
    rc = l->host.alloc(tasks_b, &h_raw);
    if (rc) return rc;
    u64* d_off = (u64*)d_raw;
    MTask* d_tasks = (MTask*)((char*)d_raw + off_b);
    u64* d_status = (u64*)((char*)d_raw + off_b + tasks_b);
    // patch symbolic offsets (index+1 encoded in the pointer) into device addresses
    MTask* ht = (MTask*)h_raw;
    size_t ti = 0;
    for (int lv = 0; lv < levels; ++lv)
        for (MTask T : plan[lv].tasks) {
            if (lv > 0) {
                T.a.off = d_off + ((uintptr_t)T.a.off - 1);
                if (T.b.base) T.b.off = d_off + ((uintptr_t)T.b.off - 1);
            }
            ht[ti++] = T;
        }
    CK(cudaMemcpyAsync(d_tasks, ht, tasks_b, cudaMemcpyHostToDevice, l->stream));
    CK(cudaMemsetAsync(d_status, 0, status_b, l->stream));
    size_t tpos = 0;
    uint64_t spos = 0;
    for (int lv = 0; lv < levels; ++lv) {
        Level& L = plan[lv];
        MParams P;
        P.tasks = d_tasks + tpos;
        P.ntasks = (u32)L.tasks.size();
        P.ntiles = (u32)L.ntiles;
        P.out = L.out;
        P.out_cap = (L.out == (u64*)d_out) ? out_cap : total;
        P.out_off = d_off + L.off_index;
        P.status = d_status + spos;
        P.ticket = (u32*)(d_status + spos + L.ntiles);
        P.err = l->d_err;
        merge_kernel<<<(unsigned)L.ntiles, M_NT, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        l->launches += 1;
        g_stats.launches += 1;
        tpos += L.tasks.size();
        spos += L.ntiles + 2;
    }
    CK(cudaMemcpyAsync(d_out_len, d_off + plan[levels - 1].off_index + 1, sizeof(u64), cudaMemcpyDeviceToDevice, l->stream));
    return DGX_OK;
}

// Single-pass multiway merge (merge_multi.cuh) for 3..64 runs: msample -> merge tree over the samples -> mplan2 ->
// mmerge3 -> mscan -> mcompact.
static int merge_multi_impl(dgx_lane* l, const std::vector<MRef>& runs, const std::vector<uint64_t>& ub, uint64_t total,
                            uint64_t* d_out, size_t out_cap, uint64_t* d_out_len) {
    const size_t k = runs.size();
    // about one sample per 512 values, shared among the runs in proportion to their lengths
    const uint64_t ntarget = std::min<uint64_t>(std::max<uint64_t>(total / 512, 1), uint64_t(1) << 24);
    std::vector<u32> soff(k + 1, 0);
    for (size_t j = 0; j < k; ++j) soff[j + 1] = soff[j] + (u32)((unsigned __int128)ub[j] * ntarget / total);
    const u32 nsamp = soff[k];
    void *h_raw, *d_raw;
    const size_t runs_b = k * sizeof(MRef), soff_b = (k + 1) * sizeof(u32);
    int rc = l->host.alloc(runs_b + soff_b, &h_raw);
    if (rc) return rc;
    memcpy(h_raw, runs.data(), runs_b);
    memcpy((char*)h_raw + runs_b, soff.data(), soff_b);
    const size_t a_samples = ((runs_b + soff_b + 255) & ~size_t(255));
    const size_t a_split = a_samples + (size_t)(nsamp + 1) * 8;
    const size_t a_nsplit = a_split + (size_t)(nsamp + 1) * 8;
    const size_t a_bounds = a_nsplit + 256;
    const size_t a_tin = a_bounds + (size_t)(nsamp + 2) * k * 8;
    const size_t a_tout = a_tin + (size_t)(nsamp + 2) * 8;
    const size_t a_tcnt = a_tout + (size_t)(nsamp + 3) * 8;
    const size_t a_tlo = ((a_tcnt + (size_t)(nsamp + 2) * 4 + 255) & ~size_t(255));
    const size_t a_end = a_tlo + (size_t)(nsamp + 2) * 8;
    rc = l->ws.alloc(a_end, &d_raw);
    if (rc) return rc;
    void* d_scratch;
    rc = l->ws.alloc(total * sizeof(u64), &d_scratch);
    if (rc) return rc;
    char* d = (char*)d_raw;
    CK(cudaMemcpyAsync(d, h_raw, runs_b + soff_b, cudaMemcpyHostToDevice, l->stream));
    MMParams P;
    P.runs = (const MRef*)d;
    P.k = (u32)k;
    P.samp_off = (const u32*)(d + runs_b);
    P.nsamp = nsamp;
    P.samples = (u64*)(d + a_samples);
    P.splitters = (u64*)(d + a_split);
    P.nsplit = (const u64*)(d + a_nsplit);
    const u32 max_tiles = nsamp / MM_STRIDE + 1;
    P.bounds = (u64*)(d + a_bounds);
    P.nbs = max_tiles + 1;
    P.tile_in = (u64*)(d + a_tin);
    P.tile_cnt = (u32*)(d + a_tcnt);
    P.tile_out = (u64*)(d + a_tout);
    P.tile_lo = (u64*)(d + a_tlo);
    P.scratch = (u64*)d_scratch;
    P.out = (u64*)d_out;
    P.out_cap = out_cap;
    P.out_len = (u64*)d_out_len;
    P.err = l->d_err;
    P.ahead = 3u * (u32)g_num_sms;  // the tile the same SM slot most likely runs next: 3 resident CTAs per SM
    if (nsamp) {
        msample_kernel<<<(nsamp + 255) / 256, 256, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        l->launches += 1;
        g_stats.launches += 1;
        // the sample runs are sorted: the merge tree (with de-duplication) yields the distinct splitters
        std::vector<MRef> sruns;
        std::vector<uint64_t> sub;
        for (size_t j = 0; j < k; ++j) {
            const u32 sj = soff[j + 1] - soff[j];
            if (!sj) continue;
            sruns.push_back(MRef{P.samples + soff[j], nullptr, (u64)sj});
            sub.push_back(sj);
        }
        rc = merge_tree_impl(l, sruns, sub, nsamp, (uint64_t*)P.splitters, nsamp, (uint64_t*)(d + a_nsplit));
        if (rc) return rc;
    } else {
        CK(cudaMemsetAsync(d + a_nsplit, 0, 8, l->stream));
    }
    const uint64_t nb = (uint64_t)P.nbs * k;
    mplan2_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    mmerge3_kernel<<<max_tiles, T_NT, T_SMEM, l->stream>>>(P);
    CK(cudaGetLastError());
    mscan_kernel<<<1, 1024, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    mcompact_kernel<<<max_tiles, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    l->launches += 4;
    g_stats.launches += 4;
    return DGX_OK;
}

extern "C" int dgx_dev_merge_sorted(dgx_lane* l, const uint64_t* const* d_lists, const size_t* lens, size_t k,
                                    uint64_t* d_out, size_t out_cap, uint64_t* d_out_len) {
    if (!l) return fail(DGX_ERR_ARG, "null lane");
    if (int rc = lane_begin_op(l)) return rc;
    std::vector<ListDesc> ld(k);
    for (size_t i = 0; i < k; ++i) ld[i] = {d_lists[i], lens[i], nullptr};
    g_stats.calls += 1;
    const int rc = merge_sorted_impl(l, ld.data(), k, d_out, out_cap, d_out_len);
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_out_len, sizeof(uint64_t));
    return rc;
}

// ---------------------------------------------------------------------------
// UidPack decode, device level
// ---------------------------------------------------------------------------
struct dgx_dev_pack {
    DPack pk;
    void* d_mem = nullptr;
    size_t bytes = 0;
    size_t exact_len = 0;
    uint32_t block_size = 0;
};

// Device layout of a pack: [base u64 | delta_off u64 (n+1) | uid_off u64 (n+1) | num u32 | pad to 16]
// followed by the delta bytes (16-byte aligned, 48 readable bytes of slack for the 16-byte TMA granule and
// the 17-byte group reads).  The metadata image is assembled in pinned staging memory so that a pack
// crosses PCIe as TWO copies (metadata, deltas) and the k packs of a query as 1 + k: small copies cost
// several microseconds of DMA set-up each and used to outweigh the bytes.
struct PackLayout {
    size_t nb, dbytes, o_doff, o_uoff, o_num, meta_bytes, dpad;
};
static PackLayout pack_layout(const dgx_pack_view* v) {
    PackLayout L;
    L.nb = v ? v->nblocks : 0;
    L.dbytes = L.nb ? (size_t)v->delta_off[L.nb] : 0;
    L.o_doff = L.nb * 8;
    L.o_uoff = L.o_doff + (L.nb + 1) * 8;
    L.o_num = L.o_uoff + (L.nb + 1) * 8;
    L.meta_bytes = (L.o_num + L.nb * 4 + 15) & ~size_t(15);
    L.dpad = ((L.dbytes + 15) & ~size_t(15)) + 48;
    return L;
}
// The block-table walk of every staging route: writes uid_off[0..nb] (exclusive prefix of NumUids, every block's
// output offset) and returns ExactLen and the largest NumUids.  The kernels trust the block table: offsets must
// ascend and every block must hold at least the 5-byte minimum of each group its NumUids needs (ceil((n-1)/4),
// codec.go:76-96).  A pack that fails this is refused (the shim stays on the Go path) instead of being walked.
static int walk_block_table(const dgx_pack_view* v, uint64_t* uid_off, uint64_t* exact_len, uint32_t* max_num_out) {
    const size_t nb = v ? v->nblocks : 0;
    uint64_t acc = 0;
    uint32_t max_num = 0;
    for (size_t i = 0; i < nb; ++i) {
        uid_off[i] = acc;
        const uint32_t num = v->num_uids[i];
        acc += num;
        max_num = std::max(max_num, num);
        const uint64_t b0 = v->delta_off[i], b1 = v->delta_off[i + 1];
        const uint64_t need = num > 1 ? 5ull * ((uint64_t)(num + 2) / 4) : 0;
        if (b1 < b0 || b1 - b0 < need)
            return fail(DGX_ERR_ARG, "malformed UidPack: block %zu has %lld delta bytes, NumUids %u needs >= %llu",
                        i, (long long)(b1 - b0), num, (unsigned long long)need);
    }
    uid_off[nb] = acc;
    *exact_len = acc;
    *max_num_out = max_num;
    return DGX_OK;
}

// The pack v (nullptr: the empty pack) at the device addresses of its arrays.  sysmem: the arrays other than uid_off
// are mapped pinned host memory.  d_mem: the allocation the pack owns (nullptr: workspace or host memory).
static dgx_dev_pack dev_pack(const dgx_pack_view* v, uint64_t exact_len, uint32_t max_num, const void* base,
                             const void* delta_off, const void* num, const void* deltas, const void* uid_off, bool sysmem,
                             size_t bytes, void* d_mem) {
    dgx_dev_pack P;
    P.pk.nblocks = v ? v->nblocks : 0;
    P.pk.base = (const u64*)base;
    P.pk.delta_off = (const u64*)delta_off;
    P.pk.uid_off = (const u64*)uid_off;
    P.pk.num = (const u32*)num;
    P.pk.deltas = (const unsigned char*)deltas;
    P.pk.max_num = max_num;
    P.pk.sysmem = sysmem ? 1 : 0;
    P.d_mem = d_mem;
    P.bytes = bytes;
    P.exact_len = exact_len;
    P.block_size = v ? v->block_size : 0;
    return P;
}

// Writes v's metadata image at h (L.meta_bytes) and sets *out to the pack it becomes once that image is copied to
// d_meta and the delta bytes to d_deltas.
static int pack_fill_meta(const dgx_pack_view* v, const PackLayout& L, char* h, char* d_meta, char* d_deltas,
                          void* d_mem, dgx_dev_pack* out) {
    const size_t nb = L.nb;
    uint64_t exact = 0;
    uint32_t max_num = 0;
    int rc = walk_block_table(v, (uint64_t*)(h + L.o_uoff), &exact, &max_num);
    if (rc) return rc;
    if (nb) {
        memcpy(h, v->base, nb * 8);
        memcpy(h + L.o_doff, v->delta_off, (nb + 1) * 8);
        memcpy(h + L.o_num, v->num_uids, nb * 4);
    } else {
        memset(h + L.o_doff, 0, 8);
    }
    *out = dev_pack(v, exact, max_num, d_meta, d_meta + L.o_doff, d_meta + L.o_num, d_deltas, d_meta + L.o_uoff, false,
                    L.meta_bytes + L.dpad, d_mem);
    return DGX_OK;
}

// One pack -> its own cudaMalloc allocation (cache entries, dgx_dev_pack_upload).
static int pack_upload_owned(dgx_lane* l, const dgx_pack_view* v, dgx_dev_pack* out) {
    const PackLayout L = pack_layout(v);
    const size_t total = L.meta_bytes + L.dpad;
    void* d_mem = nullptr;
    cudaError_t e = cudaMalloc(&d_mem, total);
    if (e != cudaSuccess) return fail(DGX_ERR_OOM, "cudaMalloc(%zu) failed: %s", total, cudaGetErrorString(e));
    out->d_mem = d_mem;  // owned by *out from here on, also when a later step fails
    void* h_raw;
    int rc = l->host.alloc(L.meta_bytes, &h_raw);
    if (rc) return rc;
    char* d = (char*)d_mem;
    rc = pack_fill_meta(v, L, (char*)h_raw, d, d + L.meta_bytes, d_mem, out);
    if (rc) return rc;
    CK(cudaMemcpyAsync(d, h_raw, L.meta_bytes, cudaMemcpyHostToDevice, l->stream));
    if (L.dbytes) CK(cudaMemcpyAsync(d + L.meta_bytes, v->deltas, L.dbytes, cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += L.meta_bytes + L.dbytes;
    return DGX_OK;
}

// Device-usable alias of a pinned (cudaMallocHost / cudaHostRegister'ed, mapped) host pointer, or nullptr.
static const void* mapped_host_ptr(const void* p) {
    if (!p) return nullptr;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    if (at.type != cudaMemoryTypeHost || !at.devicePointer) return nullptr;
    return at.devicePointer;
}

// Zero-copy form of packs_upload_ws: when every array of every pack is pinned host memory the decode kernel
// reads base / NumUids / delta_off / deltas directly over PCIe; only uid_off (computed here while the block table
// is validated) is copied, one small transfer for the whole call.  Returns DGX_OK with *done = false when some
// array is pageable (the caller then stages through DMA copies).
static int packs_map_ws(dgx_lane* l, const dgx_pack_view* const* views, size_t k, dgx_dev_pack* outs, bool* done) {
    *done = false;
    if (!g_zero_copy) return DGX_OK;
    struct Dev { const void *base, *num, *doff, *del; };
    std::vector<Dev> dv(k);
    size_t uoff_total = 0;
    for (size_t i = 0; i < k; ++i) {
        const dgx_pack_view* v = views[i];
        if (!v) continue;
        if (v->nblocks == 0) return DGX_OK;  // empty views carry no arrays: take the generic path
        dv[i] = {mapped_host_ptr(v->base), mapped_host_ptr(v->num_uids), mapped_host_ptr(v->delta_off), mapped_host_ptr(v->deltas)};
        if (!dv[i].base || !dv[i].num || !dv[i].doff || !dv[i].del) return DGX_OK;
        if ((reinterpret_cast<uintptr_t>(dv[i].del) & 15u) || (reinterpret_cast<uintptr_t>(dv[i].base) & 7u) ||
            (reinterpret_cast<uintptr_t>(dv[i].doff) & 7u) || (reinterpret_cast<uintptr_t>(dv[i].num) & 3u))
            return DGX_OK;
        uoff_total += (v->nblocks + 1) * sizeof(uint64_t);
    }
    if (uoff_total == 0) return DGX_OK;
    void *d_raw, *h_raw;
    int rc = l->ws.alloc(uoff_total, &d_raw);
    if (rc) return rc;
    rc = l->host.alloc(uoff_total, &h_raw);
    if (rc) return rc;
    size_t o = 0;
    for (size_t i = 0; i < k; ++i) {
        const dgx_pack_view* v = views[i];
        if (!v) continue;
        const size_t nb = v->nblocks;
        uint64_t exact = 0;
        uint32_t max_num = 0;
        rc = walk_block_table(v, (uint64_t*)((char*)h_raw + o), &exact, &max_num);
        if (rc) return rc;
        outs[i] = dev_pack(v, exact, max_num, dv[i].base, dv[i].doff, dv[i].num, dv[i].del, (char*)d_raw + o, true, 0,
                           nullptr);
        o += (nb + 1) * sizeof(uint64_t);
        // the bytes still cross PCIe, as reads issued by the decode kernel
        g_stats.h2d += nb * 20 + (nb + 1) * 8 + (size_t)v->delta_off[nb];
    }
    CK(cudaMemcpyAsync(d_raw, h_raw, uoff_total, cudaMemcpyHostToDevice, l->stream));
    *done = true;
    return DGX_OK;
}

// Flat image of a pack (dgx_pack_image_size / dgx_pack_image_view): [base u64 x nb | delta_off u64 x (nb+1) |
// num_uids u32 x nb | pad to 16 | deltas | pad to 16].  A shim that flattens pb.UidPack.Blocks into pinned staging
// memory writes this directly; images written back to back travel as ONE DMA transfer.
static size_t image_meta_bytes(size_t nb) { return (size_t)pack_image_meta_bytes(nb); }
static bool view_is_image(const dgx_pack_view* v) {
    const size_t nb = v->nblocks;
    const char* b = (const char*)v->base;
    if (!b || (reinterpret_cast<uintptr_t>(b) & 15u)) return false;
    return (const char*)v->delta_off == b + nb * 8 && (const char*)v->num_uids == b + nb * 8 + (nb + 1) * 8 &&
           (const char*)v->deltas == b + image_meta_bytes(nb);
}
static size_t view_image_bytes(const dgx_pack_view* v) {
    return image_meta_bytes(v->nblocks) + (((size_t)v->delta_off[v->nblocks] + 15) & ~size_t(15));
}
// All packs of the call are images laid out back to back: one copy for the images, one for the uid_off tables.
static int packs_upload_run(dgx_lane* l, const dgx_pack_view* const* views, size_t k, dgx_dev_pack* outs, bool* done) {
    *done = false;
    const char* start = nullptr;
    const char* next = nullptr;
    size_t uoff_bytes = 0;
    for (size_t i = 0; i < k; ++i) {
        const dgx_pack_view* v = views[i];
        if (!v) continue;
        if (v->nblocks == 0 || !view_is_image(v)) return DGX_OK;
        if (!start) start = (const char*)v->base;
        else if ((const char*)v->base != next) return DGX_OK;
        next = (const char*)v->base + view_image_bytes(v);
        uoff_bytes += (v->nblocks + 1) * sizeof(uint64_t);
    }
    if (!start) return DGX_OK;
    const size_t run = (size_t)(next - start);
    void *d_img, *d_uoff, *h_uoff;
    int rc = l->ws.alloc(run + 64, &d_img);
    if (rc) return rc;
    rc = l->ws.alloc(uoff_bytes, &d_uoff);
    if (rc) return rc;
    rc = l->host.alloc(uoff_bytes, &h_uoff);
    if (rc) return rc;
    size_t uo = 0;
    for (size_t i = 0; i < k; ++i) {
        const dgx_pack_view* v = views[i];
        if (!v) continue;
        const size_t nb = v->nblocks;
        uint64_t exact = 0;
        uint32_t max_num = 0;
        rc = walk_block_table(v, (uint64_t*)((char*)h_uoff + uo), &exact, &max_num);
        if (rc) return rc;
        const char* d = (const char*)d_img + ((const char*)v->base - start);
        outs[i] = dev_pack(v, exact, max_num, d, d + nb * 8, d + nb * 8 + (nb + 1) * 8, d + image_meta_bytes(nb),
                           (char*)d_uoff + uo, false, view_image_bytes(v), nullptr);
        uo += (nb + 1) * sizeof(uint64_t);
    }
    CK(cudaMemcpyAsync(d_img, start, run, cudaMemcpyHostToDevice, l->stream));
    CK(cudaMemcpyAsync(d_uoff, h_uoff, uoff_bytes, cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += run + uoff_bytes;
    *done = true;
    return DGX_OK;
}

// The one way one-shot packs reach the lane's workspace: the k packs of one call, as one run of images when they
// are laid out that way, else one copy for all metadata images and one per pack for its delta bytes (straight
// from the caller's memory).  views[i] == nullptr entries are skipped.
static int packs_upload_ws(dgx_lane* l, const dgx_pack_view* const* views, size_t k, dgx_dev_pack* outs) {
    {
        bool done = false;
        int rc0 = packs_upload_run(l, views, k, outs, &done);
        if (rc0 || done) return rc0;
    }
    std::vector<PackLayout> Ls(k);
    size_t meta_total = 0, del_total = 0;
    for (size_t i = 0; i < k; ++i) {
        if (!views[i]) continue;
        Ls[i] = pack_layout(views[i]);
        meta_total += Ls[i].meta_bytes;
        del_total += Ls[i].dpad;
    }
    if (meta_total == 0) return DGX_OK;
    void *d_raw, *h_raw;
    int rc = l->ws.alloc(meta_total + del_total, &d_raw);
    if (rc) return rc;
    rc = l->host.alloc(meta_total, &h_raw);
    if (rc) return rc;
    char* d_meta = (char*)d_raw;
    char* d_del = (char*)d_raw + meta_total;
    char* h = (char*)h_raw;
    size_t mo = 0, dof = 0;
    for (size_t i = 0; i < k; ++i) {
        if (!views[i]) continue;
        rc = pack_fill_meta(views[i], Ls[i], h + mo, d_meta + mo, d_del + dof, nullptr, &outs[i]);
        if (rc) return rc;
        mo += Ls[i].meta_bytes;
        dof += Ls[i].dpad;
    }
    CK(cudaMemcpyAsync(d_meta, h, meta_total, cudaMemcpyHostToDevice, l->stream));
    for (size_t i = 0; i < k; ++i)
        if (views[i] && Ls[i].dbytes)
            CK(cudaMemcpyAsync((void*)outs[i].pk.deltas, views[i]->deltas, Ls[i].dbytes, cudaMemcpyHostToDevice, l->stream));
    for (size_t i = 0; i < k; ++i)
        if (views[i]) g_stats.h2d += Ls[i].meta_bytes + Ls[i].dbytes;
    return DGX_OK;
}

extern "C" int dgx_dev_pack_upload(dgx_lane* l, const dgx_pack_view* v, dgx_dev_pack** out) {
    if (!l || !out) return fail(DGX_ERR_ARG, "null argument");
    CK(cudaSetDevice(l->device));
    dgx_dev_pack* pk = new dgx_dev_pack();
    int rc = pack_upload_owned(l, v, pk);
    // the pinned uid_off staging must outlive the async copy
    if (rc == DGX_OK && cudaStreamSynchronize(l->stream) != cudaSuccess) rc = fail(DGX_ERR_CUDA, "pack upload failed");
    if (rc) { dgx_dev_pack_free(pk); return rc; }
    *out = pk;
    return DGX_OK;
}
extern "C" void dgx_dev_pack_free(dgx_dev_pack* pk) {
    if (!pk) return;
    if (pk->d_mem) cudaFree(pk->d_mem);
    delete pk;
}
// ExactLen of a pack, 0 when it is nil: read from a staged pack, or summed from the block counts of a ref's host view.
static uint64_t exact_len(const dgx_dev_pack* pk) { return pk ? pk->exact_len : 0; }
static uint64_t exact_len(const dgx_pack_ref& ref) {
    const dgx_pack_view* p = ref.pack;
    uint64_t n = 0;
    for (size_t b = 0; p && b < p->nblocks; ++b) n += p->num_uids[b];
    return n;
}
extern "C" size_t dgx_dev_pack_exact_len(const dgx_dev_pack* pk) { return exact_len(pk); }
extern "C" size_t dgx_dev_pack_bytes(const dgx_dev_pack* pk) { return pk ? pk->bytes : 0; }

static int decode_impl(dgx_lane* l, const DPack& pk, uint64_t seek, uint64_t* d_out, size_t out_cap,
                       uint64_t* d_out_len) {
    void* d_seek;
    int rc = l->ws.alloc(sizeof(DSeek), &d_seek);
    if (rc) return rc;
    decode_seek_kernel<<<1, 32, 0, l->stream>>>(pk, seek, (DSeek*)d_seek, (u64*)d_out_len, out_cap, l->d_err);
    CK(cudaGetLastError());
    l->launches += 1;
    g_stats.launches += 1;
    if (pk.nblocks) {
        const uint64_t warps = (pk.nblocks + D_BPW - 1) / D_BPW;
        const uint64_t ctas = (warps + D_WARPS - 1) / D_WARPS;
        decode_kernel<<<(unsigned)ctas, D_NT, sizeof(DWarpSmem) * D_WARPS, l->stream>>>(pk, (const DSeek*)d_seek, (u64*)d_out, out_cap);
        CK(cudaGetLastError());
        l->launches += 1;
        g_stats.launches += 1;
    }
    return DGX_OK;
}

extern "C" int dgx_dev_decode(dgx_lane* l, const dgx_dev_pack* pk, uint64_t seek, uint64_t* d_out, size_t out_cap,
                              uint64_t* d_out_len) {
    if (!l || !pk) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    g_stats.uids_in += pk->exact_len;
    const int rc = decode_impl(l, pk->pk, seek, d_out, out_cap, d_out_len);
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_out_len, sizeof(uint64_t));
    return rc;
}

// ---------------------------------------------------------------------------
// host-pointer entry points
// ---------------------------------------------------------------------------
// Lanes of the host-pointer entry points.  The pool is bounded: at most kMaxLanes lanes exist (each keeps a stream,
// its workspace and pinned staging at their high-water mark), a caller beyond that waits for one to come back --
// hundreds of cgo goroutines cannot pin hundreds of arenas in HBM.  A lane whose workspace grew past kLaneTrimBytes is
// shrunk when it is returned (it is idle then: every host-pointer call ends with a stream sync).
constexpr size_t kMaxLanes = 32;
constexpr size_t kLaneTrimBytes = size_t(4) << 30;
struct LaneLease {
    dgx_lane* l = nullptr;
    int rc = DGX_OK;
    LaneLease() {
        rc = dgx_init(-1);
        if (rc) return;
        bool create = false;
        {
            std::unique_lock<std::mutex> lk(g_mu);
            g_pool_cv.wait(lk, [] { return !g_pool.empty() || g_lanes_total < kMaxLanes; });
            if (!g_pool.empty()) { l = g_pool.back(); g_pool.pop_back(); }
            else { create = true; g_lanes_total += 1; }
            g_lanes_out += 1;
        }
        if (create) {
            l = dgx_lane_create(g_device, nullptr);
            if (!l) {
                rc = fail(DGX_ERR_CUDA, "cannot create lane: %s", g_err.c_str());
                std::lock_guard<std::mutex> lk(g_mu);
                g_lanes_total -= 1;
                g_lanes_out -= 1;
                g_pool_cv.notify_all();
                return;
            }
        }
        cudaSetDevice(l->device);
        l->ws.reset();
    }
    ~LaneLease() {
        if (!l) return;
        if (l->ws.cap > kLaneTrimBytes) {  // idle (synchronised) lane: give a one-off large workspace back
            cudaStreamSynchronize(l->stream);
            l->ws.destroy();
        }
        std::lock_guard<std::mutex> lk(g_mu);
        g_pool.push_back(l);
        g_lanes_out -= 1;
        g_pool_cv.notify_all();
    }
};

static int upload_list(dgx_lane* l, const uint64_t* h, size_t n, uint64_t** d) {
    void* p;
    int rc = l->ws.alloc((n + 2) * sizeof(uint64_t), &p);
    if (rc) return rc;
    if (n) CK(cudaMemcpyAsync(p, h, n * sizeof(uint64_t), cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += n * sizeof(uint64_t);
    *d = (uint64_t*)p;
    return DGX_OK;
}

// Result to the host in ONE round trip when it is short: the length word and the first kSpecHead
// values (fewer if the device buffer is smaller) are copied speculatively before the sync; only a
// longer result pays a second copy for its tail.  d_cap = values allocated behind d_out.
static int finish_to_host(dgx_lane* l, const uint64_t* d_len, const uint64_t* d_out, size_t d_cap, uint64_t* out,
                          size_t out_cap, size_t* out_len) {
    const size_t head = std::min(std::min(d_cap, out_cap), kSpecHead);
    CK(cudaMemcpyAsync(l->h_word, d_len, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (head) CK(cudaMemcpyAsync(l->h_head, d_out, head * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    int rc = dgx_lane_sync(l);
    if (rc) return rc;
    const uint64_t n = l->h_word[0];
    if (n > out_cap) return fail(DGX_ERR_CAP, "result (%llu) does not fit out_cap (%zu)", (unsigned long long)n, out_cap);
    if (n) memcpy(out, l->h_head, std::min<size_t>(n, head) * sizeof(uint64_t));
    if (n > head) {
        CK(cudaMemcpyAsync(out + head, d_out + head, (n - head) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaStreamSynchronize(l->stream));
    }
    g_stats.d2h += std::max<uint64_t>(n, head) * sizeof(uint64_t) + 8;
    g_stats.uids_out += n;
    if (out_len) *out_len = (size_t)n;
    return DGX_OK;
}

// CSR result of a batch to the host: the npairs + 1 offsets, then the values they count.
static int batch_to_host(dgx_lane* l, const void* d_out, const void* d_off, size_t npairs, uint64_t* out,
                         uint64_t* out_off, size_t out_cap) {
    CK(cudaMemcpyAsync(out_off, d_off, (npairs + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    int rc = dgx_lane_sync(l);
    if (rc) return rc;
    const uint64_t n = out_off[npairs];
    if (n > out_cap) return fail(DGX_ERR_CAP, "batch result (%llu) does not fit out_cap (%zu)", (unsigned long long)n, out_cap);
    if (n) {
        CK(cudaMemcpyAsync(out, d_out, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaStreamSynchronize(l->stream));
    }
    g_stats.d2h += (n + npairs + 1) * sizeof(uint64_t);
    g_stats.uids_out += n;
    return DGX_OK;
}

// The CSR epilogue of a host-pointer batch call: room for `cap` values (and the two a kernel may pad with) and nrows + 1
// offsets in the lane's workspace, filled by run(d_out, d_off), then copied back by batch_to_host.
template <class Run>
static int csr_to_host(dgx_lane* l, size_t cap, size_t nrows, uint64_t* out, uint64_t* out_off, size_t out_cap, Run run) {
    uint64_t *d_out, *d_off;
    WsCarve ws(l);
    ws.plain(&d_out, cap + 2);
    ws.plain(&d_off, nrows + 1);
    if (int rc = ws.commit()) return rc;
    if (int rc = run(d_out, d_off)) return rc;
    return batch_to_host(l, d_out, d_off, nrows, out, out_off, out_cap);
}

static int filter_host(int op, const uint64_t* const* lists, const size_t* lens, size_t k, uint64_t* out,
                       size_t out_cap, size_t* out_len) {
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    std::vector<ListDesc> ld(k);
    size_t cap = SIZE_MAX;
    for (size_t i = 0; i < k; ++i) {
        uint64_t* d;
        int rc = upload_list(l, lists[i], lens[i], &d);
        if (rc) return rc;
        ld[i] = {d, lens[i], nullptr};
        if (op == DGX_OP_INTERSECT) cap = std::min(cap, lens[i]);
    }
    if (op == DGX_OP_DIFFERENCE) cap = lens[0];
    void *d_out, *d_off;
    int rc = l->ws.alloc((cap + 2) * sizeof(uint64_t), &d_out);
    if (rc) return rc;
    rc = l->ws.alloc(2 * sizeof(uint64_t), &d_off);
    if (rc) return rc;
    const size_t k_off[2] = {0, k};
    rc = filter_batch_impl(l, op, ld.data(), k_off, 1, (uint64_t*)d_out, cap, (uint64_t*)d_off);
    if (rc) return rc;
    return finish_to_host(l, (uint64_t*)d_off + 1, (uint64_t*)d_out, cap, out, out_cap, out_len);
}

extern "C" int dgx_intersect2(const uint64_t* u, size_t n, const uint64_t* v, size_t m, uint64_t* out,
                              size_t out_cap, size_t* out_len) {
    const uint64_t* lists[2] = {u, v};
    const size_t lens[2] = {n, m};
    return filter_host(DGX_OP_INTERSECT, lists, lens, 2, out, out_cap, out_len);
}

extern "C" int dgx_intersect_sorted(const uint64_t* const* lists, const size_t* lens, size_t k, uint64_t* out,
                                    size_t out_cap, size_t* out_len) {
    if (k == 0) {  // IntersectSorted of no lists is the empty list (algo/uidlist.go:298-300)
        if (out_len) *out_len = 0;
        return DGX_OK;
    }
    return filter_host(DGX_OP_INTERSECT, lists, lens, k, out, out_cap, out_len);
}

extern "C" int dgx_difference(const uint64_t* u, size_t n, const uint64_t* v, size_t m, uint64_t* out,
                              size_t out_cap, size_t* out_len) {
    const uint64_t* lists[2] = {u, v};
    const size_t lens[2] = {n, m};
    return filter_host(DGX_OP_DIFFERENCE, lists, lens, 2, out, out_cap, out_len);
}

extern "C" int dgx_merge_sorted(const uint64_t* const* lists, const size_t* lens, size_t k, uint64_t* out,
                                size_t out_cap, size_t* out_len) {
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    std::vector<ListDesc> ld(k);
    size_t total = 0;
    for (size_t i = 0; i < k; ++i) {
        if (lists[i] == nullptr || lens[i] == 0) { ld[i] = {nullptr, 0, nullptr}; continue; }
        uint64_t* d;
        int rc = upload_list(l, lists[i], lens[i], &d);
        if (rc) return rc;
        ld[i] = {d, lens[i], nullptr};
        total += lens[i];
    }
    void *d_out, *d_len;
    int rc = l->ws.alloc((total + 2) * sizeof(uint64_t), &d_out);
    if (rc) return rc;
    rc = l->ws.alloc(64, &d_len);
    if (rc) return rc;
    rc = merge_sorted_impl(l, ld.data(), k, (uint64_t*)d_out, total, (uint64_t*)d_len);
    if (rc) return rc;
    return finish_to_host(l, (uint64_t*)d_len, (uint64_t*)d_out, total, out, out_cap, out_len);
}

extern "C" int dgx_intersect_batch(const uint64_t* a, const uint64_t* a_off, const uint64_t* b,
                                   const uint64_t* b_off, size_t npairs, uint64_t* out, uint64_t* out_off,
                                   size_t out_cap) {
    if (npairs == 0) { if (out_off) out_off[0] = 0; return DGX_OK; }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    const size_t na = a_off[npairs] - a_off[0], nbv = b_off[npairs] - b_off[0];
    uint64_t *d_a, *d_b;
    int rc = upload_list(l, a + a_off[0], na, &d_a);
    if (rc) return rc;
    rc = upload_list(l, b + b_off[0], nbv, &d_b);
    if (rc) return rc;
    std::vector<ListDesc> ld(2 * npairs);
    std::vector<size_t> k_off(npairs + 1);
    size_t cap = 0;
    for (size_t i = 0; i < npairs; ++i) {
        const size_t la = a_off[i + 1] - a_off[i], lb = b_off[i + 1] - b_off[i];
        ld[2 * i] = {d_a + (a_off[i] - a_off[0]), la, nullptr};
        ld[2 * i + 1] = {d_b + (b_off[i] - b_off[0]), lb, nullptr};
        k_off[i] = 2 * i;
        cap += std::min(la, lb);
    }
    k_off[npairs] = 2 * npairs;
    return csr_to_host(l, cap, npairs, out, out_off, out_cap, [&](uint64_t* d_out, uint64_t* d_off) {
        return filter_batch_impl(l, DGX_OP_INTERSECT, ld.data(), k_off.data(), npairs, d_out, cap, d_off);
    });
}

extern "C" int dgx_decode(const dgx_pack_view* p, uint64_t seek, uint64_t* out, size_t out_cap, size_t* out_len) {
    if (!p || p->nblocks == 0) {  // nil / empty pack decodes to the empty list (codec/codec.go:445-446)
        if (out_len) *out_len = 0;
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    dgx_dev_pack pk;
    int rc = packs_upload_ws(l, &p, 1, &pk);
    if (rc) return rc;
    g_stats.uids_in += pk.exact_len;
    void *d_out, *d_len;
    rc = l->ws.alloc((pk.exact_len + 2) * sizeof(uint64_t), &d_out);
    if (rc) return rc;
    rc = l->ws.alloc(64, &d_len);
    if (rc) return rc;
    rc = decode_impl(l, pk.pk, seek, (uint64_t*)d_out, pk.exact_len, (uint64_t*)d_len);
    if (rc) return rc;
    return finish_to_host(l, (uint64_t*)d_len, (uint64_t*)d_out, pk.exact_len, out, out_cap, out_len);
}

extern "C" int dgx_decode_intersect_sorted(const dgx_pack_view* p, uint64_t seek, const uint64_t* const* lists,
                                           const size_t* lens, size_t k, uint64_t* out, size_t out_cap,
                                           size_t* out_len) {
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    std::vector<ListDesc> ld(k + 1);
    int rc;
    size_t cap = SIZE_MAX;
    for (size_t i = 0; i < k; ++i) {
        uint64_t* d;
        rc = upload_list(l, lists[i], lens[i], &d);
        if (rc) return rc;
        ld[i + 1] = {d, lens[i], nullptr};
        cap = std::min(cap, lens[i]);
    }
    void *d_dec = nullptr, *d_len;
    rc = l->ws.alloc(64, &d_len);
    if (rc) return rc;
    size_t exact = 0;
    if (p && p->nblocks) {
        dgx_dev_pack pk;
        rc = packs_upload_ws(l, &p, 1, &pk);
        if (rc) return rc;
        exact = pk.exact_len;
        rc = l->ws.alloc((exact + 2) * sizeof(uint64_t), &d_dec);
        if (rc) return rc;
        rc = decode_impl(l, pk.pk, seek, (uint64_t*)d_dec, exact, (uint64_t*)d_len);
        if (rc) return rc;
    } else {
        rc = l->ws.alloc(16, &d_dec);
        if (rc) return rc;
        CK(cudaMemsetAsync(d_len, 0, 8, l->stream));
    }
    g_stats.uids_in += exact;
    ld[0] = {(const uint64_t*)d_dec, exact, (const uint64_t*)d_len};
    cap = std::min(cap, exact);
    void *d_out, *d_off;
    rc = l->ws.alloc((cap + 2) * sizeof(uint64_t), &d_out);
    if (rc) return rc;
    rc = l->ws.alloc(2 * sizeof(uint64_t), &d_off);
    if (rc) return rc;
    const size_t k_off[2] = {0, k + 1};
    rc = filter_batch_impl(l, DGX_OP_INTERSECT, ld.data(), k_off, 1, (uint64_t*)d_out, cap, (uint64_t*)d_off);
    if (rc) return rc;
    return finish_to_host(l, (uint64_t*)d_off + 1, (uint64_t*)d_out, cap, out, out_cap, out_len);
}

// algo.IntersectCompressedWith on the device (compressed_kernel.cuh): v-ranges of the blocks, decode +
// probe of the touched blocks in shared memory, order-preserving compaction of v.
static int icw_impl(dgx_lane* l, const dgx_dev_pack& pk, uint64_t after, const uint64_t* d_v, size_t m,
                    uint64_t* d_out, size_t out_cap, uint64_t* d_len) {
    const size_t nb = pk.pk.nblocks;
    if (nb == 0 || m == 0) {
        CK(cudaMemsetAsync(d_len, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    const size_t tiles = (m + CP_TILE - 1) / CP_TILE;
    IcwParams P;
    CompactParams C;
    WsCarve ws(l);
    ws.zeroed(&P.vlo, nb);
    ws.zeroed(&P.vhi, nb);
    ws.zeroed(&P.keep, m);
    ws.zeroed(&C.status, tiles);
    ws.zeroed(&C.ticket, 16);
    if (int rc = ws.commit()) return rc;
    P.pk = pk.pk;
    P.v = (const u64*)d_v;
    P.m = m;
    P.after = after;
    // search the shorter side's elements in the longer side (the reference's linVsBinRatio idea, :49-59)
    if (m < nb) icw_ranges_by_v_kernel<<<(unsigned)((m + 255) / 256), 256, 0, l->stream>>>(P);
    else icw_ranges_by_block_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    const uint64_t warps = (nb + D_BPW - 1) / D_BPW;
    icw_probe_kernel<<<(unsigned)((warps + D_WARPS - 1) / D_WARPS), D_NT, sizeof(DWarpSmem) * D_WARPS, l->stream>>>(P);
    CK(cudaGetLastError());
    C.v = (const u64*)d_v;
    C.keep = P.keep;
    C.m = m;
    C.out = (u64*)d_out;
    C.out_cap = out_cap;
    C.out_len = (u64*)d_len;
    C.err = l->d_err;
    compact_kernel<<<(unsigned)tiles, CP_NT, 0, l->stream>>>(C);
    CK(cudaGetLastError());
    l->launches += 3;
    g_stats.launches += 3;
    g_stats.uids_in += pk.exact_len + m;
    return DGX_OK;
}

static int intersect_compressed_host(const dgx_pack_ref& ref, uint64_t after_uid, const uint64_t* v, size_t m,
                                     uint64_t* out, size_t out_cap, size_t* out_len);

extern "C" int dgx_intersect_compressed(const dgx_pack_view* p, uint64_t after_uid, const uint64_t* v, size_t m,
                                        uint64_t* out, size_t out_cap, size_t* out_len) {
    const dgx_pack_ref ref = {p, 0, 0};
    return intersect_compressed_host(ref, after_uid, v, m, out, out_cap, out_len);
}
extern "C" int dgx_intersect_compressed_ref(const dgx_pack_ref* ref, uint64_t after_uid, const uint64_t* v, size_t m,
                                            uint64_t* out, size_t out_cap, size_t* out_len) {
    if (!ref) return fail(DGX_ERR_ARG, "null ref");
    return intersect_compressed_host(*ref, after_uid, v, m, out, out_cap, out_len);
}

// ---------------------------------------------------------------------------
// HBM-resident pack cache + IntersectSorted over packs
// ---------------------------------------------------------------------------
// Production holds posting lists as UidPacks (posting.List.plist.Pack, posting/list.go:1795-1800) and
// decodes them per query.  Here a pack crosses PCIe compressed (about 1.5 B/UID instead of 8) and is
// expanded on the device; a pack the caller names with (key, version) -- immutable bytes, e.g. the hash
// of its Badger key and the commit timestamp of the layer -- stays in HBM in its compressed form and
// later calls skip the copy.  Eviction is LRU by bytes; entries in use by a running call are pinned.
static size_t pack_device_bytes(const dgx_pack_view* v) {
    const PackLayout L = pack_layout(v);
    return L.meta_bytes + L.dpad;
}

struct CacheKey {
    uint64_t key, version;
    bool operator==(const CacheKey& o) const { return key == o.key && version == o.version; }
};
struct CacheKeyHash {
    size_t operator()(const CacheKey& k) const {
        uint64_t h = k.key * 0x9E3779B97F4A7C15ull ^ (k.version + 0x7F4A7C15ull + (k.key << 6) + (k.key >> 2));
        return (size_t)(h ^ (h >> 29));
    }
};
struct CacheEntry {
    CacheKey id;
    dgx_dev_pack pk;
    cudaEvent_t ready = nullptr;  // recorded after the upload: other streams wait on it before reading
    int refs = 0;
    std::list<CacheEntry*>::iterator lru;
};
static std::mutex g_cache_mu;
static std::unordered_map<CacheKey, CacheEntry*, CacheKeyHash> g_cache;
static std::list<CacheEntry*> g_cache_lru;  // front = most recently used
static size_t g_cache_bytes = 0;
static size_t g_cache_max = size_t(16) << 30;  // DGX_CACHE_BYTES / dgx_cache_configure (a fifth of an 80 GB H100)
static bool g_cache_env_read = false;
static dgx_cache_stats g_cache_stats = {0, 0, 0, 0, 0, 0};

static void cache_free_entry(CacheEntry* e) {
    // refs == 0: every call that used the entry has synchronised its stream, nothing queued reads it
    if (e->pk.d_mem) cudaFree(e->pk.d_mem);
    if (e->ready) cudaEventDestroy(e->ready);
    g_cache_bytes -= e->pk.bytes;
    delete e;
}
// g_cache_mu held.  Drops least-recently-used idle entries until `extra` more bytes fit.
static void cache_make_room(size_t extra) {
    auto it = g_cache_lru.end();
    while (g_cache_bytes + extra > g_cache_max && it != g_cache_lru.begin()) {
        --it;
        CacheEntry* e = *it;
        if (e->refs > 0) continue;
        it = g_cache_lru.erase(it);
        g_cache.erase(e->id);
        cache_free_entry(e);
        g_cache_stats.evictions += 1;
    }
}

extern "C" int dgx_cache_configure(size_t max_bytes) {
    std::lock_guard<std::mutex> lk(g_cache_mu);
    g_cache_env_read = true;
    g_cache_max = max_bytes;
    cache_make_room(0);
    return DGX_OK;
}
extern "C" void dgx_cache_clear(void) {
    std::lock_guard<std::mutex> lk(g_cache_mu);
    const size_t keep = g_cache_max;
    g_cache_max = 0;
    cache_make_room(0);
    g_cache_max = keep;
}
extern "C" void dgx_cache_get_stats(dgx_cache_stats* out) {
    if (!out) return;
    std::lock_guard<std::mutex> lk(g_cache_mu);
    *out = g_cache_stats;
    out->bytes = g_cache_bytes;
    out->entries = g_cache.size();
    out->max_bytes = g_cache_max;
}

// The packs of one host-pointer call on lane `l`.  pk[i] is refs[i]'s pack: the empty pack for a nil or empty ref,
// the cached copy for a named ref (one reference held until the set is destroyed), else copied into the lane's
// workspace together with the call's other one-shot packs.  Declared after the call's LaneLease, so that it is
// destroyed first: unless the call reported synced() after its final host sync, the destructor synchronises the
// lane stream before it drops the references, since queued work may still read the cached packs.
struct PackSet {
    std::vector<dgx_dev_pack> pk;
    int rc = DGX_OK;
    // zero_copy: pinned one-shot packs are decoded in place when DGX_ZERO_COPY=1 (packs_map_ws)
    PackSet(dgx_lane* lane, const dgx_pack_ref* refs, size_t k, bool zero_copy = false) : pk(k), l(lane) {
        std::vector<const dgx_pack_view*> oneshot(k, nullptr);
        for (size_t i = 0; i < k; ++i) {
            const dgx_pack_view* v = refs[i].pack;
            if (!v || v->nblocks == 0) continue;
            CacheEntry* e = nullptr;
            if (refs[i].key) rc = acquire(refs[i], &e);
            if (rc) return;
            if (e) pk[i] = e->pk;
            else oneshot[i] = v;
        }
        bool mapped = false;
        if (zero_copy) rc = packs_map_ws(l, oneshot.data(), k, pk.data(), &mapped);
        if (rc == DGX_OK && !mapped) rc = packs_upload_ws(l, oneshot.data(), k, pk.data());
    }
    // &pk[i] for every i: the row table of the *_rows impls
    std::vector<const dgx_dev_pack*> rows() const {
        std::vector<const dgx_dev_pack*> r(pk.size());
        for (size_t i = 0; i < pk.size(); ++i) r[i] = &pk[i];
        return r;
    }
    // rc of the call's final step, which ends in a host sync when it succeeds
    int synced(int call_rc) {
        finished = call_rc == DGX_OK;
        return call_rc;
    }
    ~PackSet() {
        if (!finished) cudaStreamSynchronize(l->stream);
        if (held.empty()) return;
        std::lock_guard<std::mutex> lk(g_cache_mu);
        for (CacheEntry* e : held) e->refs -= 1;
    }

  private:
    dgx_lane* l;
    std::vector<CacheEntry*> held;
    bool finished = false;

    // *out: the cache entry holding ref's pack, one reference taken; nullptr when the pack does not fit (cache
    // disabled, pack larger than the cache, everything pinned) and is copied for this call only.
    int acquire(const dgx_pack_ref& ref, CacheEntry** out) {
        const dgx_pack_view* v = ref.pack;
        std::lock_guard<std::mutex> lk(g_cache_mu);
        if (!g_cache_env_read) {
            g_cache_env_read = true;
            if (const char* s = getenv("DGX_CACHE_BYTES")) g_cache_max = (size_t)strtoull(s, nullptr, 10);
        }
        const CacheKey id{ref.key, ref.version};
        auto it = g_cache.find(id);
        if (it != g_cache.end()) {
            CacheEntry* e = it->second;
            e->refs += 1;
            held.push_back(e);
            g_cache_lru.erase(e->lru);
            g_cache_lru.push_front(e);
            e->lru = g_cache_lru.begin();
            g_cache_stats.hits += 1;
            CK(cudaStreamWaitEvent(l->stream, e->ready, 0));
            *out = e;
            return DGX_OK;
        }
        g_cache_stats.misses += 1;
        const size_t bytes = pack_device_bytes(v);
        if (bytes > g_cache_max) return DGX_OK;
        cache_make_room(bytes);
        if (g_cache_bytes + bytes > g_cache_max) return DGX_OK;
        CacheEntry* e = new CacheEntry();
        e->id = id;
        // the enqueue (a handful of async copies) happens under the lock so that a second caller
        // asking for the same pack finds the recorded event, never a half-built entry
        int rc = pack_upload_owned(l, v, &e->pk);
        if (rc == DGX_OK && (cudaEventCreateWithFlags(&e->ready, cudaEventDisableTiming) != cudaSuccess ||
                             cudaEventRecord(e->ready, l->stream) != cudaSuccess))
            rc = fail(DGX_ERR_CUDA, "cache event failed");
        if (rc) {
            if (e->pk.d_mem) cudaFree(e->pk.d_mem);
            if (e->ready) cudaEventDestroy(e->ready);
            delete e;
            return rc;
        }
        e->refs = 1;
        held.push_back(e);
        g_cache_bytes += e->pk.bytes;
        g_cache_lru.push_front(e);
        e->lru = g_cache_lru.begin();
        g_cache.emplace(id, e);
        *out = e;
        return DGX_OK;
    }
};

// Decode every pack of `pks` in full, side by side, with one launch; d_lists[i] receives pack i.
static int decode_batch_impl(dgx_lane* l, const dgx_dev_pack* pks, size_t k, uint64_t** d_lists) {
    void *h_raw, *d_raw;
    int rc = l->host.alloc(k * sizeof(DJob), &h_raw);
    if (rc) return rc;
    rc = l->ws.alloc(k * sizeof(DJob), &d_raw);
    if (rc) return rc;
    DJob* hj = (DJob*)h_raw;
    u64 warps = 0;
    u32 nj = 0;
    for (size_t i = 0; i < k; ++i) {
        void* d;
        rc = l->ws.alloc((pks[i].exact_len + 2) * sizeof(uint64_t), &d);
        if (rc) return rc;
        d_lists[i] = (uint64_t*)d;
        if (pks[i].pk.nblocks == 0) continue;
        hj[nj].pk = pks[i].pk;
        hj[nj].out = (u64*)d;
        hj[nj].warp_base = warps;
        warps += (pks[i].pk.nblocks + D_BPW - 1) / D_BPW;
        ++nj;
        g_stats.uids_in += pks[i].exact_len;
    }
    if (nj == 0) return DGX_OK;
    CK(cudaMemcpyAsync(d_raw, h_raw, nj * sizeof(DJob), cudaMemcpyHostToDevice, l->stream));
    const u64 ctas = (warps + D_WARPS - 1) / D_WARPS;
    if (ctas > 0x7fffffffull) return fail(DGX_ERR_ARG, "packs too large for one decode launch");
    decode_batch_kernel<<<(unsigned)ctas, D_NT, sizeof(DWarpSmem) * D_WARPS, l->stream>>>((const DJob*)d_raw, nj, warps);
    CK(cudaGetLastError());
    l->launches += 1;
    g_stats.launches += 1;
    return DGX_OK;
}

extern "C" int dgx_intersect_sorted_packed(const dgx_pack_ref* refs, size_t k, uint64_t* out, size_t out_cap,
                                           size_t* out_len) {
    if (out_len) *out_len = 0;
    if (k == 0) return DGX_OK;  // IntersectSorted of no lists (algo/uidlist.go:298-300)
    if (!refs) return fail(DGX_ERR_ARG, "null refs");
    for (size_t i = 0; i < k; ++i)  // a nil / empty pack decodes to the empty list: the intersection is empty
        if (!refs[i].pack || refs[i].pack->nblocks == 0) return DGX_OK;
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    PackSet ps(l, refs, k, /*zero_copy=*/true);
    if (ps.rc) return ps.rc;
    std::vector<uint64_t*> d_lists(k, nullptr);
    int rc = decode_batch_impl(l, ps.pk.data(), k, d_lists.data());
    if (rc) return rc;
    std::vector<ListDesc> ld(k);
    size_t cap = SIZE_MAX;
    for (size_t i = 0; i < k; ++i) {
        ld[i] = {d_lists[i], ps.pk[i].exact_len, nullptr};
        cap = std::min(cap, ps.pk[i].exact_len);
    }
    void *d_out, *d_off;
    rc = l->ws.alloc((cap + 2) * sizeof(uint64_t), &d_out);
    if (rc) return rc;
    rc = l->ws.alloc(2 * sizeof(uint64_t), &d_off);
    if (rc) return rc;
    const size_t k_off[2] = {0, k};
    rc = filter_batch_impl(l, DGX_OP_INTERSECT, ld.data(), k_off, 1, (uint64_t*)d_out, cap, (uint64_t*)d_off);
    if (rc) return rc;
    return ps.synced(finish_to_host(l, (uint64_t*)d_off + 1, (uint64_t*)d_out, cap, out, out_cap, out_len));
}

static int intersect_compressed_host(const dgx_pack_ref& ref, uint64_t after_uid, const uint64_t* v, size_t m,
                                     uint64_t* out, size_t out_cap, size_t* out_len) {
    if (out_len) *out_len = 0;
    if (ref.pack == nullptr) return DGX_OK;  // `if pack == nil { return }` (algo/uidlist.go:34-36): o is left untouched
    if (m >= (size_t(1) << 32)) {             // v-ranges are 32-bit: beyond that, decode from the seek and filter
        const uint64_t* lists[1] = {v};
        const size_t lens[1] = {m};
        return dgx_decode_intersect_sorted(ref.pack, after_uid, lists, lens, 1, out, out_cap, out_len);
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    PackSet ps(l, &ref, 1);
    if (ps.rc) return ps.rc;
    uint64_t* d_v;
    int rc = upload_list(l, v, m, &d_v);
    if (rc) return rc;
    void *d_out, *d_len;
    rc = l->ws.alloc((m + 2) * sizeof(uint64_t), &d_out);
    if (rc) return rc;
    rc = l->ws.alloc(64, &d_len);
    if (rc) return rc;
    rc = icw_impl(l, ps.pk[0], after_uid, d_v, m, (uint64_t*)d_out, m, (uint64_t*)d_len);
    if (rc) return rc;
    return ps.synced(finish_to_host(l, (uint64_t*)d_len, (uint64_t*)d_out, m, out, out_cap, out_len));
}

// Decoder.Seek / SeekToBlock / LinearSeek / Next / UnpackBlock for one call (codec/codec.go:154-384), on the device.
extern "C" int dgx_pack_seek(const dgx_pack_view* p, int kind, uint64_t uid, int whence, size_t block_idx,
                             uint64_t* out, size_t out_cap, size_t* out_len, size_t* block_idx_after) {
    if (out_len) *out_len = 0;
    if (block_idx_after) *block_idx_after = 0;
    if (!p || p->nblocks == 0) return DGX_OK;  // nil pack: every seek returns an empty slice
    if (kind < SK_SEEK || kind > SK_UNPACK || (whence != 0 && whence != 1)) return fail(DGX_ERR_ARG, "bad seek kind / whence");
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    dgx_dev_pack pk;
    int rc = packs_upload_ws(l, &p, 1, &pk);
    if (rc) return rc;
    void *d_out, *d_meta;
    const size_t cap = std::max<size_t>(pk.pk.max_num, 1);
    rc = l->ws.alloc((cap + 2) * sizeof(uint64_t), &d_out);
    if (rc) return rc;
    rc = l->ws.alloc(64, &d_meta);
    if (rc) return rc;
    SeekParams S;
    S.pk = pk.pk;
    S.uid = uid;
    S.whence = whence;
    S.kind = kind;
    S.block_idx = block_idx;
    S.out = (u64*)d_out;
    S.out_meta = (u64*)d_meta;
    pack_seek_kernel<<<1, 32, 0, l->stream>>>(S);
    CK(cudaGetLastError());
    l->launches += 1;
    g_stats.launches += 1;
    CK(cudaMemcpyAsync(l->h_word, d_meta, 2 * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(l->h_head, d_out, std::min(cap, kSpecHead) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    rc = dgx_lane_sync(l);
    if (rc) return rc;
    const uint64_t n = l->h_word[0];
    if (block_idx_after) *block_idx_after = (size_t)l->h_word[1];
    if (n > out_cap) return fail(DGX_ERR_CAP, "block (%llu uids) does not fit out_cap (%zu)", (unsigned long long)n, out_cap);
    if (n > kSpecHead) {
        CK(cudaMemcpyAsync(out, d_out, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaStreamSynchronize(l->stream));
    } else if (n) {
        memcpy(out, l->h_head, n * sizeof(uint64_t));
    }
    if (out_len) *out_len = (size_t)n;
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// codec.Encode on the device, packed set operations
// ---------------------------------------------------------------------------
extern "C" size_t dgx_pack_image_size(size_t nblocks, size_t delta_bytes) {
    return image_meta_bytes(nblocks) + ((delta_bytes + 15) & ~size_t(15));
}
extern "C" int dgx_pack_image_view(void* image, uint32_t block_size, size_t nblocks, size_t delta_bytes, dgx_pack_view* view) {
    (void)delta_bytes;
    if (!image || !view || (reinterpret_cast<uintptr_t>(image) & 15u)) return fail(DGX_ERR_ARG, "image must be 16-byte aligned");
    char* b = (char*)image;
    view->block_size = block_size;
    view->nblocks = nblocks;
    view->base = (const uint64_t*)b;
    view->delta_off = (const uint64_t*)(b + nblocks * 8);
    view->num_uids = (const uint32_t*)(b + nblocks * 8 + (nblocks + 1) * 8);
    view->deltas = (const uint8_t*)(b + image_meta_bytes(nblocks));
    return DGX_OK;
}

extern "C" void dgx_encode_bound(size_t n, uint32_t block_size, size_t* nblocks_cap, size_t* delta_cap) {
    const size_t B = block_size ? block_size : 1;
    // a sorted list crosses a multiple of 2^32 rarely: room for 64 extra (short) blocks; dgx_encode reports sizes
    // that suffice with DGX_ERR_CAP when a list has more upper-word changes than that, so one retry succeeds
    const size_t nb = n ? (n + B - 1) / B + 64 : 0;
    if (nblocks_cap) *nblocks_cap = nb;
    if (delta_cap) *delta_cap = 17 * (n / 4 + nb + 1);  // every group is at most 17 bytes
}

struct EncOut {           // device arrays of one encoded pack (workspace memory)
    u64* base; u32* num; u64* delta_off; unsigned char* deltas; u64* counts;
    size_t n, nblocks_cap, delta_cap;  // n: most uids encoded (the list's length when it is read from the device)
};
// Encodes d_u[0..n) (n from *d_n when d_n != nullptr, at most n) into workspace arrays.
static int encode_impl(dgx_lane* l, const uint64_t* d_u, size_t n, const uint64_t* d_n, uint32_t block_size,
                       size_t nblocks_cap, size_t delta_cap, EncOut* out) {
    const size_t tiles_a = std::max<size_t>(1, (n + EN_TILE - 1) / EN_TILE);
    const size_t tiles_b = std::max<size_t>(1, (nblocks_cap + EN_TILE - 1) / EN_TILE);
    const size_t seg_cap = std::min<size_t>(n, nblocks_cap) + 2;  // more segments than blocks cannot fit anyway
    EncParams P;
    WsCarve ws(l);
    ws.zeroed(&P.counts, 8);
    ws.zeroed(&P.ticket, 8);
    ws.zeroed(&P.err, 8);
    ws.zeroed(&P.status, tiles_a + tiles_b);
    ws.plain(&P.seg_start, seg_cap);
    ws.plain(&P.seg_blk, seg_cap);
    ws.plain(&P.base, nblocks_cap + 1);
    ws.plain(&P.blk_start, nblocks_cap + 1);
    ws.plain(&P.blk_bytes, nblocks_cap + 1);
    ws.plain(&P.delta_off, nblocks_cap + 1);
    ws.plain(&P.num, nblocks_cap + 1 + 16);
    ws.plain(&P.deltas, delta_cap + 64);
    if (int rc = ws.commit()) return rc;
    P.u = (const u64*)d_u;
    P.n = n;
    P.n_dyn = (const u64*)d_n;
    P.bsz = block_size ? block_size : 1;
    u64* status_b = P.status + tiles_a;
    P.seg_cap = seg_cap;
    P.nblocks_cap = nblocks_cap;
    P.delta_cap = delta_cap;
    // a list with more segments than seg_cap cannot be encoded into nblocks_cap blocks: the segment pass would
    // overrun its array, so it is bounded by the same capacity check (segments <= blocks)
    enc_segments_kernel<<<(unsigned)tiles_a, EN_NT, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    enc_segscan_kernel<<<1, 1024, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    const size_t warp_ctas = std::max<size_t>(1, (nblocks_cap * 32 + 255) / 256);
    enc_sizes_kernel<<<(unsigned)warp_ctas, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)tiles_b, EN_NT, 0, l->stream>>>(P.blk_bytes, P.delta_off, P.counts + 1, nblocks_cap, status_b,
                                                               P.ticket + 1, P.counts + 2);
    CK(cudaGetLastError());
    enc_write_kernel<<<(unsigned)warp_ctas, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    l->launches += 5;
    g_stats.launches += 5;
    out->base = P.base; out->num = P.num; out->delta_off = P.delta_off; out->deltas = P.deltas; out->counts = P.counts;
    out->n = n; out->nblocks_cap = nblocks_cap; out->delta_cap = delta_cap;
    return DGX_OK;
}

// counts + arrays of an encoded pack to the caller's arrays.  *nblocks / *delta_bytes: capacity in, size out.
static int encode_to_host(dgx_lane* l, const EncOut& E, uint32_t block_size, uint64_t* base, uint32_t* num_uids,
                          uint64_t* delta_off, uint8_t* deltas, size_t* nblocks, size_t* delta_bytes, dgx_pack_view* view) {
    CK(cudaMemcpyAsync(l->h_word, E.counts, 3 * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    int rc = dgx_lane_sync(l);
    if (rc) return rc;
    const uint64_t nb = l->h_word[1];
    // the deltas are sized only when the blocks fit; otherwise the call again needs room for the most that nb blocks
    // of n uids can take (every group is at most 17 bytes), so that it does not fail a second time on the deltas
    const uint64_t db = nb > E.nblocks_cap ? 17 * (E.n / 4 + nb + 1) : l->h_word[2];
    const size_t cap_nb = *nblocks, cap_db = *delta_bytes;
    *nblocks = (size_t)nb;
    *delta_bytes = (size_t)db;
    if (nb > cap_nb || nb > E.nblocks_cap || db > cap_db || db > E.delta_cap)
        return fail(DGX_ERR_CAP, "pack needs %llu blocks / %llu delta bytes (given %zu / %zu): sizes returned, call again",
                    (unsigned long long)nb, (unsigned long long)db, cap_nb, cap_db);
    if (nb) {
        CK(cudaMemcpyAsync(base, E.base, nb * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaMemcpyAsync(num_uids, E.num, nb * sizeof(uint32_t), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaMemcpyAsync(delta_off, E.delta_off, (nb + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
        if (db) CK(cudaMemcpyAsync(deltas, E.deltas, db, cudaMemcpyDeviceToHost, l->stream));
        CK(cudaStreamSynchronize(l->stream));
    } else if (delta_off) {
        delta_off[0] = 0;
    }
    g_stats.d2h += nb * 20 + db + 32;
    if (view) {
        view->block_size = block_size;
        view->nblocks = (size_t)nb;
        view->base = base;
        view->num_uids = num_uids;
        view->delta_off = delta_off;
        view->deltas = deltas;
    }
    return DGX_OK;
}

extern "C" int dgx_encode(const uint64_t* uids, size_t n, uint32_t block_size, uint64_t* base, uint32_t* num_uids,
                          uint64_t* delta_off, uint8_t* deltas, size_t* nblocks, size_t* delta_bytes, dgx_pack_view* view) {
    if (!nblocks || !delta_bytes) return fail(DGX_ERR_ARG, "null capacity arguments");
    if (n == 0) {  // Encoder.Done without Add: the nil pack (codec/codec.go:125-136)
        *nblocks = 0; *delta_bytes = 0;
        if (view) { view->block_size = block_size; view->nblocks = 0; view->base = base; view->num_uids = num_uids; view->delta_off = delta_off; view->deltas = deltas; }
        if (delta_off) delta_off[0] = 0;
        return DGX_OK;
    }
    if (!uids || !base || !num_uids || !delta_off || !deltas) return fail(DGX_ERR_ARG, "null argument");
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += n;
    uint64_t* d_u;
    int rc = upload_list(l, uids, n, &d_u);
    if (rc) return rc;
    EncOut E;
    rc = encode_impl(l, d_u, n, nullptr, block_size, *nblocks, *delta_bytes, &E);
    if (rc) return rc;
    return encode_to_host(l, E, block_size, base, num_uids, delta_off, deltas, nblocks, delta_bytes, view);
}

// algo.IntersectWithLinPacked / DifferencePacked / MergeSortedPacked (algo/packed.go:35-297) by composition on
// the device: decode the operands side by side, run the plain-list kernel, encode the result -- operands and
// result cross PCIe compressed and nothing decoded leaves the device.  The reference's block-at-a-time loops
// have three behaviours its own tests never reach (oracle/packed.py, DESIGN section 5: IntersectSortedPacked
// keeps only ls[0] ∩ ls[1], DifferencePacked's handling of v running out of blocks); these entry points compute
// the set operation the function names, which is what every case of algo/packed_test.go expects.
static int packed_op_host(int kind /*0 intersect, 1 difference, 2 merge*/, const dgx_pack_ref* refs, size_t k,
                          uint32_t block_size, uint64_t* base, uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas,
                          size_t* nblocks, size_t* delta_bytes, dgx_pack_view* view) {
    if (!nblocks || !delta_bytes) return fail(DGX_ERR_ARG, "null capacity arguments");
    if (k && !refs) return fail(DGX_ERR_ARG, "null refs");
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    PackSet ps(l, refs, k);
    if (ps.rc) return ps.rc;
    std::vector<uint64_t*> d_lists(k, nullptr);
    int rc = decode_batch_impl(l, ps.pk.data(), k, d_lists.data());
    if (rc) return rc;
    std::vector<ListDesc> ld(k);
    size_t mn = SIZE_MAX, total = 0;
    for (size_t i = 0; i < k; ++i) {
        ld[i] = {d_lists[i], ps.pk[i].exact_len, nullptr};
        mn = std::min(mn, ps.pk[i].exact_len);
        total += ps.pk[i].exact_len;
    }
    const size_t cap = kind == 0 ? (k ? mn : 0) : (kind == 1 ? (k ? ps.pk[0].exact_len : 0) : total);
    void *d_out, *d_off, *d_len;
    rc = l->ws.alloc((cap + 2) * sizeof(uint64_t), &d_out);
    if (rc) return rc;
    rc = l->ws.alloc(64, &d_off);
    if (rc) return rc;
    if (kind == 2) {
        d_len = d_off;
        rc = merge_sorted_impl(l, ld.data(), k, (uint64_t*)d_out, cap, (uint64_t*)d_len);
    } else if (k == 0) {
        d_len = d_off;
        CK(cudaMemsetAsync(d_len, 0, 8, l->stream));
    } else {
        const size_t k_off[2] = {0, k};
        rc = filter_batch_impl(l, kind == 0 ? DGX_OP_INTERSECT : DGX_OP_DIFFERENCE, ld.data(), k_off, 1,
                               (uint64_t*)d_out, cap, (uint64_t*)d_off);
        d_len = (uint64_t*)d_off + 1;
    }
    if (rc) return rc;
    size_t nb_cap, db_cap;
    dgx_encode_bound(cap, block_size, &nb_cap, &db_cap);
    nb_cap = std::max(nb_cap, std::min(*nblocks, cap));  // a larger capacity from the caller is honoured
    db_cap = std::max(db_cap, 17 * (cap / 4 + nb_cap + 1));  // and room for the deltas of that many blocks
    EncOut E;
    rc = encode_impl(l, (const uint64_t*)d_out, cap, (const uint64_t*)d_len, block_size, nb_cap, db_cap, &E);
    if (rc) return rc;
    return ps.synced(encode_to_host(l, E, block_size, base, num_uids, delta_off, deltas, nblocks, delta_bytes, view));
}

extern "C" int dgx_intersect_packed(const dgx_pack_ref* u, const dgx_pack_ref* v, uint32_t block_size, uint64_t* base,
                                    uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas, size_t* nblocks,
                                    size_t* delta_bytes, dgx_pack_view* view) {
    if (!u || !v) return fail(DGX_ERR_ARG, "null ref");
    const dgx_pack_ref refs[2] = {*u, *v};
    return packed_op_host(0, refs, 2, block_size, base, num_uids, delta_off, deltas, nblocks, delta_bytes, view);
}
extern "C" int dgx_difference_packed(const dgx_pack_ref* u, const dgx_pack_ref* v, uint32_t block_size, uint64_t* base,
                                     uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas, size_t* nblocks,
                                     size_t* delta_bytes, dgx_pack_view* view) {
    if (!u || !v) return fail(DGX_ERR_ARG, "null ref");
    const dgx_pack_ref refs[2] = {*u, *v};
    return packed_op_host(1, refs, 2, block_size, base, num_uids, delta_off, deltas, nblocks, delta_bytes, view);
}
extern "C" int dgx_merge_sorted_packed(const dgx_pack_ref* refs, size_t k, uint32_t block_size, uint64_t* base,
                                       uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas, size_t* nblocks,
                                       size_t* delta_bytes, dgx_pack_view* view) {
    return packed_op_host(2, refs, k, block_size, base, num_uids, delta_off, deltas, nblocks, delta_bytes, view);
}
extern "C" int dgx_intersect_sorted_packed_out(const dgx_pack_ref* refs, size_t k, uint32_t block_size, uint64_t* base,
                                               uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas, size_t* nblocks,
                                               size_t* delta_bytes, dgx_pack_view* view) {
    return packed_op_host(0, refs, k, block_size, base, num_uids, delta_off, deltas, nblocks, delta_bytes, view);
}

// ---------------------------------------------------------------------------
// IndexOf batch, shared-list batch
// ---------------------------------------------------------------------------
extern "C" int dgx_index_of_batch(const uint64_t* u, size_t n, const uint64_t* uids, size_t m, int64_t* idx) {
    if (m == 0) return DGX_OK;
    if (!uids || !idx || (n && !u)) return fail(DGX_ERR_ARG, "null argument");
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    uint64_t *d_u, *d_q;
    void* d_idx;
    int rc = upload_list(l, u, n, &d_u);
    if (rc) return rc;
    rc = upload_list(l, uids, m, &d_q);
    if (rc) return rc;
    rc = l->ws.alloc(m * sizeof(int64_t), &d_idx);
    if (rc) return rc;
    const unsigned blocks = (unsigned)std::min<uint64_t>((m + 255) / 256, (uint64_t)g_num_sms * 16);
    index_of_kernel<<<blocks, 256, 0, l->stream>>>((const u64*)d_u, (u64)n, (const u64*)d_q, (u64)m, (long long*)d_idx);
    CK(cudaGetLastError());
    l->launches += 1;
    g_stats.launches += 1;
    g_stats.uids_in += n + m;
    CK(cudaMemcpyAsync(idx, d_idx, m * sizeof(int64_t), cudaMemcpyDeviceToHost, l->stream));
    g_stats.d2h += m * sizeof(int64_t);
    return dgx_lane_sync(l);
}

extern "C" int dgx_intersect_batch_shared(const uint64_t* a, const uint64_t* a_off, size_t npairs, const uint64_t* b,
                                          size_t m, uint64_t* out, uint64_t* out_off, size_t out_cap) {
    if (npairs == 0) { if (out_off) out_off[0] = 0; return DGX_OK; }
    if (!a_off || !out_off) return fail(DGX_ERR_ARG, "null argument");
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    const size_t na = a_off[npairs] - a_off[0];
    uint64_t *d_a, *d_b;
    int rc = upload_list(l, a + a_off[0], na, &d_a);
    if (rc) return rc;
    rc = upload_list(l, b, m, &d_b);  // the shared list crosses PCIe once
    if (rc) return rc;
    std::vector<ListDesc> ld(2 * npairs);
    std::vector<size_t> k_off(npairs + 1);
    size_t cap = 0;
    for (size_t i = 0; i < npairs; ++i) {
        const size_t la = a_off[i + 1] - a_off[i];
        ld[2 * i] = {d_a + (a_off[i] - a_off[0]), la, nullptr};
        ld[2 * i + 1] = {d_b, m, nullptr};
        k_off[i] = 2 * i;
        cap += std::min(la, m);
    }
    k_off[npairs] = 2 * npairs;
    return csr_to_host(l, cap, npairs, out, out_off, out_cap, [&](uint64_t* d_out, uint64_t* d_off) {
        return filter_batch_impl(l, DGX_OP_INTERSECT, ld.data(), k_off.data(), npairs, d_out, cap, d_off);
    });
}

// ---------------------------------------------------------------------------
// IntersectCompressedWith over many packs (handleUidPostings)
// ---------------------------------------------------------------------------
// Row i = algo.IntersectCompressedWith(packs[i], after, v) for every row with six launches whatever nrows is
// (compressed_kernel.cuh): ranges, slot sizes, slot scan, probe, count scan, gather.  Workspace: ~44 bytes per
// block of the batch plus a slot buffer of sum_i min(m, ExactLen_i) values.
static int icw_rows_impl(dgx_lane* l, const dgx_dev_pack* const* packs, size_t nrows, uint64_t after, const uint64_t* d_v,
                         size_t m, uint64_t* d_out, size_t out_cap, uint64_t* d_out_off) {
    if (m >= (size_t(1) << 32)) return fail(DGX_ERR_ARG, "v has %zu uids: per-block v-ranges are 32-bit", m);
    size_t nj = 0;
    uint64_t nb = 0, thr = 0, warps = 0, exact = 0, slots_cap = 0;
    for (size_t i = 0; i < nrows; ++i)
        if (packs[i] && packs[i]->pk.nblocks) ++nj;
    IcwRowsParams P;
    IcwJob* hj;
    uint64_t* h_rows;
    WsCarve ws(l);
    ws.copied(&P.jobs, &hj, nj);
    ws.copied(&P.row_blk, &h_rows, nrows + 1);
    if (int rc = ws.stage()) return rc;
    size_t j = 0;
    for (size_t i = 0; i < nrows; ++i) {
        h_rows[i] = nb;
        const dgx_dev_pack* p = packs[i];
        if (!p || p->pk.nblocks == 0) continue;
        const uint64_t pnb = p->pk.nblocks;
        IcwJob& J = hj[j++];
        J.pk = p->pk;
        J.blk_base = nb;
        J.thr_base = thr;
        J.warp_base = warps;
        J.by_v = pnb > m;
        nb += pnb;
        thr += J.by_v ? m : pnb;
        warps += (pnb + D_BPW - 1) / D_BPW;
        exact += p->exact_len;
        slots_cap += std::min<uint64_t>(m, p->exact_len);
    }
    h_rows[nrows] = nb;
    g_stats.uids_in += exact + m;
    if (nb == 0 || m == 0) {
        CK(cudaMemsetAsync(d_out_off, 0, (nrows + 1) * sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    const uint64_t kMaxGrid = 0x7fffffffull;
    const uint64_t g_rng = (thr + 255) / 256, g_blk = (nb + 255) / 256, tiles = (nb + EN_TILE - 1) / EN_TILE;
    const uint64_t g_probe = (warps + D_WARPS - 1) / D_WARPS, g_gather = (std::max<uint64_t>(nb * 32, nrows + 1) + 255) / 256;
    if (std::max({g_rng, g_blk, tiles, g_probe, g_gather}) > kMaxGrid || nj > 0xffffffffull)
        return fail(DGX_ERR_ARG, "batch too large for one launch (%llu blocks, %zu rows)", (unsigned long long)nb, nrows);
    u64* status;
    u32* tickets;
    ws.zeroed(&P.vlo, nb);
    ws.zeroed(&P.vhi, nb);
    ws.zeroed(&status, 2 * tiles);
    ws.zeroed(&tickets, 4);
    ws.plain(&P.slot, nb);
    ws.plain(&P.slot_off, nb + 1);
    ws.plain(&P.cnt, nb);
    ws.plain(&P.cnt_off, nb + 1);
    ws.plain(&P.slots, slots_cap);
    if (int rc = ws.commit()) return rc;
    P.njobs = (u32)nj;
    P.v = (const u64*)d_v;
    P.m = m;
    P.after = after;
    P.nblocks = nb;
    P.nthreads = thr;
    P.nwarps = warps;
    P.slots_cap = slots_cap;
    P.nrows = nrows;
    P.out = (u64*)d_out;
    P.out_cap = out_cap;
    P.out_off = (u64*)d_out_off;
    P.err = l->d_err;
    const u64* d_nb = P.row_blk + nrows;  // the block count as a device word (scan length)
    icw_rows_ranges_kernel<<<(unsigned)g_rng, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    icw_rows_slots_kernel<<<(unsigned)g_blk, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)tiles, EN_NT, 0, l->stream>>>(P.slot, P.slot_off, d_nb, nb, status, tickets, nullptr);
    CK(cudaGetLastError());
    icw_rows_probe_kernel<<<(unsigned)g_probe, D_NT, sizeof(DWarpSmem) * D_WARPS, l->stream>>>(P);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)tiles, EN_NT, 0, l->stream>>>(P.cnt, P.cnt_off, d_nb, nb, status + tiles, tickets + 1, nullptr);
    CK(cudaGetLastError());
    icw_rows_gather_kernel<<<(unsigned)g_gather, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    l->launches += 6;
    g_stats.launches += 6;
    return DGX_OK;
}

extern "C" int dgx_dev_intersect_compressed_rows(dgx_lane* l, const dgx_dev_pack* const* packs, size_t nrows,
                                                 uint64_t after_uid, const uint64_t* d_v, size_t m, uint64_t* d_out,
                                                 size_t out_cap, uint64_t* d_out_off) {
    if (!l || !d_out_off || (nrows && !packs) || (m && !d_v)) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    const int rc = icw_rows_impl(l, packs, nrows, after_uid, d_v, m, d_out, out_cap, d_out_off);
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    return rc;
}

extern "C" int dgx_intersect_compressed_rows(const dgx_pack_ref* refs, size_t nrows, uint64_t after_uid,
                                             const uint64_t* v, size_t m, uint64_t* out, uint64_t* out_off,
                                             size_t out_cap) {
    if (!out_off) return fail(DGX_ERR_ARG, "null out_off");
    if (nrows == 0) { out_off[0] = 0; return DGX_OK; }
    if (!refs || (m && !v)) return fail(DGX_ERR_ARG, "null argument");
    if (m >= (size_t(1) << 32)) return fail(DGX_ERR_ARG, "v has %zu uids: per-block v-ranges are 32-bit", m);
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    PackSet ps(l, refs, nrows);  // nil / empty packs are packs of no blocks: empty rows
    if (ps.rc) return ps.rc;
    const std::vector<const dgx_dev_pack*> rows = ps.rows();
    size_t cap = 0;
    for (const dgx_dev_pack& p : ps.pk) cap += std::min<size_t>(m, p.exact_len);
    uint64_t* d_v;
    int rc = upload_list(l, v, m, &d_v);
    if (rc) return rc;
    return ps.synced(csr_to_host(l, cap, nrows, out, out_off, out_cap, [&](uint64_t* d_out, uint64_t* d_off) {
        return icw_rows_impl(l, rows.data(), nrows, after_uid, d_v, m, d_out, cap, d_off);
    }));
}

// ---------------------------------------------------------------------------
// IntersectCompressedWith of one pack against every row of a uid matrix (intersectBucket)
// ---------------------------------------------------------------------------
// The offsets off[0 .. nrows] (host memory) of the CSR array `name` must start at 0, never decrease and total less than
// `limit`, the width the kernels count its elements in: checked before anything the offsets index is read.
static int check_offsets(const char* name, const uint64_t* off, size_t nrows, uint64_t limit) {
    if (off[0] != 0) return fail(DGX_ERR_ARG, "%s[0] is %llu, not 0", name, (unsigned long long)off[0]);
    for (size_t r = 0; r < nrows; ++r)
        if (off[r + 1] < off[r]) return fail(DGX_ERR_ARG, "%s decreases at row %zu", name, r);
    if (off[nrows] >= limit)
        return fail(DGX_ERR_ARG, "%s totals %llu: at most %llu", name, (unsigned long long)off[nrows],
                    (unsigned long long)(limit - 1));
    return DGX_OK;
}

// Row i = algo.IntersectCompressedWith(pk, 0, v[v_off[i] .. v_off[i+1])) with six launches whatever nrows, M and the
// block count are (compressed_kernel.cuh): locate, unit scan, place, probe, keep scan, gather.  Workspace: at most 36
// bytes per element of v plus about 20 per block and 8 per row.  v_off is host memory, already checked.
static int icw_matrix_impl(dgx_lane* l, const dgx_dev_pack& pk, const uint64_t* d_v, const uint64_t* v_off, size_t nrows,
                           uint64_t* d_out, size_t out_cap, uint64_t* d_out_off) {
    const uint64_t m = v_off[nrows], nb = pk.pk.nblocks;
    g_stats.uids_in += pk.exact_len + m;
    if (nb == 0 || m == 0) {  // nothing can match: every row is empty
        CK(cudaMemsetAsync(d_out_off, 0, (nrows + 1) * sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (nb > 0xffffffffull) return fail(DGX_ERR_ARG, "pack of %llu blocks: block indices are 32-bit", (unsigned long long)nb);
    uint64_t units = 0;  // units of ascending rows: each row touches at most min(|row|, nb) blocks
    for (size_t r = 0; r < nrows; ++r) units += std::min<uint64_t>(v_off[r + 1] - v_off[r], nb);
    const uint64_t kMaxGrid = 0x7fffffffull;
    const uint64_t g_elem = (m + 255) / 256, g_gather = (std::max<uint64_t>(m, nrows + 1) + 255) / 256;
    const uint64_t t_blk = (nb + EN_TILE - 1) / EN_TILE, t_elem = (m + EN_TILE - 1) / EN_TILE;
    const uint64_t g_probe = ((units + 31) / 32 + D_WARPS - 1) / D_WARPS;
    if (std::max({g_elem, g_gather, g_probe}) > kMaxGrid)
        return fail(DGX_ERR_ARG, "matrix too large for one launch (%llu uids, %zu rows)", (unsigned long long)m, nrows);
    // the copied table is [v_off | nb | m]
    IcwMatrixParams P;
    uint64_t* h_tab;
    u64* status;
    u32* tickets;
    WsCarve ws(l);
    ws.copied(&P.v_off, &h_tab, nrows + 3);
    if (int rc = ws.stage()) return rc;
    memcpy(h_tab, v_off, (nrows + 1) * sizeof(uint64_t));
    h_tab[nrows + 1] = nb;
    h_tab[nrows + 2] = m;
    ws.zeroed(&P.bcount, nb);
    ws.zeroed(&P.bfill, nb);
    ws.zeroed(&status, t_blk + t_elem);
    ws.zeroed(&tickets, 2);
    ws.zeroed(&P.bad, 1);
    ws.plain(&P.head, m);
    ws.plain(&P.boff, nb + 1);
    ws.plain(&P.unit, units);
    ws.plain(&P.keep, m);
    ws.plain(&P.kex, m + 1);
    ws.plain(&P.ublk, units);
    if (int rc = ws.commit()) return rc;
    P.pk = pk.pk;
    P.v = (const u64*)d_v;
    P.m = m;
    P.nrows = nrows;
    const u64* d_nb = P.v_off + nrows + 1;  // scan lengths as device words
    const u64* d_m = P.v_off + nrows + 2;
    P.unit_cap = units;
    P.out = (u64*)d_out;
    P.out_cap = out_cap;
    P.out_off = (u64*)d_out_off;
    P.err = l->d_err;
    icw_mx_locate_kernel<<<(unsigned)g_elem, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)t_blk, EN_NT, 0, l->stream>>>(P.bcount, P.boff, d_nb, nb, status, tickets, nullptr);
    CK(cudaGetLastError());
    icw_mx_place_kernel<<<(unsigned)g_elem, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    icw_mx_probe_kernel<<<(unsigned)g_probe, D_NT, sizeof(DWarpSmem) * D_WARPS, l->stream>>>(P);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)t_elem, EN_NT, 0, l->stream>>>(P.keep, P.kex, d_m, m, status + t_blk, tickets + 1, nullptr);
    CK(cudaGetLastError());
    icw_mx_gather_kernel<<<(unsigned)g_gather, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    l->launches += 6;
    g_stats.launches += 6;
    return DGX_OK;
}

extern "C" int dgx_dev_intersect_compressed_matrix(dgx_lane* l, const dgx_dev_pack* pk, const uint64_t* d_v,
                                                   const uint64_t* v_off, size_t nrows, uint64_t* d_out, size_t out_cap,
                                                   uint64_t* d_out_off) {
    if (!l || !d_out_off || (nrows && !v_off)) return fail(DGX_ERR_ARG, "null argument");
    static const uint64_t zero_off = 0;
    if (nrows == 0) v_off = &zero_off;
    if (int rc = check_offsets("v_off", v_off, nrows, uint64_t(1) << 32)) return rc;
    if (v_off[nrows] && !d_v) return fail(DGX_ERR_ARG, "null d_v");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    const dgx_dev_pack empty = dev_pack(nullptr, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr, false, 0, nullptr);
    const int rc = icw_matrix_impl(l, pk ? *pk : empty, d_v, v_off, nrows, d_out, out_cap, d_out_off);
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    return rc;
}

extern "C" int dgx_intersect_compressed_matrix(const dgx_pack_ref* ref, const uint64_t* v, const uint64_t* v_off,
                                               size_t nrows, uint64_t* out, uint64_t* out_off, size_t out_cap) {
    if (!out_off) return fail(DGX_ERR_ARG, "null out_off");
    if (nrows == 0) { out_off[0] = 0; return DGX_OK; }
    if (!ref || !v_off) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = check_offsets("v_off", v_off, nrows, uint64_t(1) << 32)) return rc;
    const size_t m = v_off[nrows];
    if (m && !v) return fail(DGX_ERR_ARG, "null v");
    if (!ref->pack || ref->pack->nblocks == 0) {  // nil / empty pack: every row is empty, nothing runs
        memset(out_off, 0, (nrows + 1) * sizeof(uint64_t));
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    PackSet ps(l, ref, 1);
    if (ps.rc) return ps.rc;
    size_t cap = 0;
    for (size_t r = 0; r < nrows; ++r) cap += std::min<size_t>(v_off[r + 1] - v_off[r], ps.pk[0].exact_len);
    uint64_t* d_v;
    int rc = upload_list(l, v, m, &d_v);
    if (rc) return rc;
    return ps.synced(csr_to_host(l, cap, nrows, out, out_off, out_cap, [&](uint64_t* d_out, uint64_t* d_off) {
        return icw_matrix_impl(l, ps.pk[0], d_v, v_off, nrows, d_out, cap, d_off);
    }));
}

// ---------------------------------------------------------------------------
// List.Uids over a task's keys, mutable layers included (handleUidPostings)
// ---------------------------------------------------------------------------
// The resolved mutable layers of a task's rows, as every List.Uids entry point takes them: mut_off (host memory) with
// fewer than 2^31 entries in all, so that no sum of class words carries (list_uids_kernel.cuh), and the uids and flags
// present when there are entries.
static int check_mut_layers(const uint64_t* mut_off, size_t nrows, const void* mut_uids, const void* mut_flags) {
    if (int rc = check_offsets("mut_off", mut_off, nrows, uint64_t(1) << 31)) return rc;
    if (mut_off[nrows] && (!mut_uids || !mut_flags)) return fail(DGX_ERR_ARG, "null mutable layer");
    return DGX_OK;
}

// The host forms stage the layers' nmut uids and flags in the lane's workspace, one copy each.
static int upload_mut_layers(dgx_lane* l, const uint64_t* mut_uids, const uint8_t* mut_flags, size_t nmut,
                             uint64_t** d_uids, const uint8_t** d_flags) {
    int rc = upload_list(l, mut_uids, nmut, d_uids);
    if (rc) return rc;
    void* p;
    rc = l->ws.alloc(nmut + 16, &p);
    if (rc) return rc;
    if (nmut) CK(cudaMemcpyAsync(p, mut_flags, nmut, cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += nmut;
    *d_flags = (const uint8_t*)p;
    return DGX_OK;
}

// The host-side checks of both forms, before anything is copied: m, the mutable layers, modes, and the bound that keeps
// the MaxInt32 cut of List.Uids (posting/list.go:1840, 1864-1870) from biting.  rows[i] is row i's pack.
static_assert(LU_COMPRESSED == DGX_UIDS_COMPRESSED && LU_PROBE == DGX_UIDS_PROBE && LU_ITERATE == DGX_UIDS_ITERATE &&
                  LU_DEL == DGX_MUT_DEL && LU_VALUE == DGX_MUT_VALUE,
              "list_uids_kernel.cuh reads the modes and flags of include/dgx.h");
template <class Row>
static int list_uids_check(const uint8_t* mode, size_t nrows, const uint64_t* mut_off, const void* mut_uids,
                           const void* mut_flags, size_t m, const Row* rows) {
    const uint64_t k31 = uint64_t(1) << 31;
    if (m == 0) return fail(DGX_ERR_ARG, "v is empty: an unfiltered read is not a List.Uids row call");
    if (m >= k31) return fail(DGX_ERR_ARG, "v has %zu uids: at most 2^31 - 1", m);
    if (int rc = check_mut_layers(mut_off, nrows, mut_uids, mut_flags)) return rc;
    for (size_t r = 0; r < nrows; ++r) {
        if (mode[r] > LU_ITERATE) return fail(DGX_ERR_ARG, "row %zu has mode %u", r, (unsigned)mode[r]);
        const uint64_t nm = mut_off[r + 1] - mut_off[r];
        if (mode[r] == LU_COMPRESSED && nm) return fail(DGX_ERR_ARG, "row %zu is compressed but has mutable entries", r);
        if (mode[r] == LU_ITERATE && exact_len(rows[r]) + nm >= k31)
            return fail(DGX_ERR_ARG, "iterate row %zu has %llu postings: at most 2^31 - 1", r,
                        (unsigned long long)(exact_len(rows[r]) + nm));
    }
    return DGX_OK;
}

// Row i = List.Uids of row i's branch (list_uids_kernel.cuh) with the six launches of icw_rows_impl (pack ∩ v, after 0)
// and five of its own: classify, entry scan, rows, row scan, write.  When no row has a non-empty pack, icw_rows_impl
// launches nothing and the call makes five.  mode and mut_off are host memory, already checked.
static int list_uids_impl(dgx_lane* l, const dgx_dev_pack* const* packs, const uint8_t* mode, size_t nrows,
                          const uint64_t* d_mut, const uint8_t* d_flags, const uint64_t* mut_off, uint64_t after,
                          const uint64_t* d_v, size_t m, uint64_t* d_out, size_t out_cap, uint64_t* d_out_off) {
    const uint64_t nmut = mut_off[nrows];
    uint64_t a_cap = 0;
    for (size_t i = 0; i < nrows; ++i) a_cap += std::min<uint64_t>(m, exact_len(packs[i]));
    const uint64_t kMaxGrid = 0x7fffffffull;
    const uint64_t g_mut = std::max<uint64_t>((nmut + 255) / 256, 1), g_rows = (nrows + 255) / 256;
    const uint64_t g_write = (std::max<uint64_t>(a_cap + nmut, nrows + 1) + 255) / 256;
    const uint64_t t_mut = std::max<uint64_t>((nmut + EN_TILE - 1) / EN_TILE, 1), t_rows = (nrows + EN_TILE - 1) / EN_TILE;
    if (std::max({g_mut, g_rows, g_write}) > kMaxGrid)
        return fail(DGX_ERR_ARG, "batch too large for one launch (%llu uids, %zu rows)", (unsigned long long)(a_cap + nmut),
                    nrows);
    LuParams P;
    uint64_t *h_off, *h_first, *h_len;
    const u64* d_nmut;  // scan lengths as device words: nmut, nrows
    unsigned char* h_mode;
    u64 *status, *a, *a_off;
    u32* tickets;
    WsCarve ws(l);
    ws.copied(&P.mut_off, &h_off, nrows + 1);
    ws.copied(&P.first, &h_first, nrows);
    ws.copied(&d_nmut, &h_len, 2);
    ws.copied(&P.mode, &h_mode, nrows);
    if (int rc = ws.stage()) return rc;
    memcpy(h_off, mut_off, (nrows + 1) * sizeof(uint64_t));
    for (size_t i = 0; i < nrows; ++i) {
        const bool reads_pack = mode[i] != LU_COMPRESSED && packs[i] && packs[i]->pk.nblocks;
        h_first[i] = reads_pack ? (uint64_t)(uintptr_t)packs[i]->pk.base : 0;
    }
    h_len[0] = nmut;
    h_len[1] = nrows;
    memcpy(h_mode, mode, nrows);
    ws.zeroed(&status, t_mut + t_rows);
    ws.zeroed(&tickets, 2);
    ws.zeroed(&P.bad, 1);
    ws.plain(&a, a_cap + 2);
    ws.plain(&a_off, nrows + 1);
    ws.plain(&P.cls, nmut);
    ws.plain(&P.cls_ex, nmut + 1);
    ws.plain(&P.lo, nrows);
    ws.plain(&P.cnt, nrows);
    if (int rc = ws.commit()) return rc;
    const u64* d_nrows = d_nmut + 1;
    P.nrows = nrows;
    P.mut = (const u64*)d_mut;
    P.flags = d_flags;
    P.nmut = nmut;
    P.after = after;
    P.v = (const u64*)d_v;
    P.m = m;
    P.a = a;
    P.a_off = a_off;
    P.a_cap = a_cap;
    P.out = (u64*)d_out;
    P.out_cap = out_cap;
    P.out_off = (u64*)d_out_off;
    P.err = l->d_err;
    // pack ∩ v of every row from uid 0: each mode applies its own bound afterwards
    if (int rc = icw_rows_impl(l, packs, nrows, 0, d_v, m, (uint64_t*)a, a_cap, (uint64_t*)a_off)) return rc;
    lu_classify_kernel<<<(unsigned)g_mut, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)t_mut, EN_NT, 0, l->stream>>>(P.cls, P.cls_ex, d_nmut, nmut, status, tickets, nullptr);
    CK(cudaGetLastError());
    lu_rows_kernel<<<(unsigned)g_rows, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)t_rows, EN_NT, 0, l->stream>>>(P.cnt, P.out_off, d_nrows, nrows, status + t_mut,
                                                                tickets + 1, nullptr);
    CK(cudaGetLastError());
    lu_write_kernel<<<(unsigned)g_write, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    l->launches += 5;
    g_stats.launches += 5;
    g_stats.uids_in += nmut;
    return DGX_OK;
}

extern "C" int dgx_dev_list_uids_rows(dgx_lane* l, const dgx_dev_pack* const* packs, const uint8_t* mode, size_t nrows,
                                      const uint64_t* d_mut_uids, const uint8_t* d_mut_flags, const uint64_t* mut_off,
                                      uint64_t after_uid, const uint64_t* d_v, size_t m, uint64_t* d_out,
                                      size_t out_cap, uint64_t* d_out_off) {
    if (!l || !d_out_off) return fail(DGX_ERR_ARG, "null argument");
    if (nrows == 0) {
        if (int rc = lane_begin_op(l)) return rc;
        CK(cudaMemsetAsync(d_out_off, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (!packs || !mode || !mut_off || !d_v) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = list_uids_check(mode, nrows, mut_off, d_mut_uids, d_mut_flags, m, packs)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    const int rc = list_uids_impl(l, packs, mode, nrows, d_mut_uids, d_mut_flags, mut_off, after_uid, d_v, m, d_out,
                                  out_cap, d_out_off);
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    return rc;
}

extern "C" int dgx_list_uids_rows(const dgx_pack_ref* refs, const uint8_t* mode, size_t nrows, const uint64_t* mut_uids,
                                  const uint8_t* mut_flags, const uint64_t* mut_off, uint64_t after_uid, const uint64_t* v,
                                  size_t m, uint64_t* out, uint64_t* out_off, size_t out_cap) {
    if (!out_off) return fail(DGX_ERR_ARG, "null out_off");
    if (nrows == 0) { out_off[0] = 0; return DGX_OK; }
    if (!refs || !mode || !mut_off || !v) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = list_uids_check(mode, nrows, mut_off, mut_uids, mut_flags, m, refs)) return rc;
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    PackSet ps(l, refs, nrows);  // nil / empty packs are packs of no blocks
    if (ps.rc) return ps.rc;
    const std::vector<const dgx_dev_pack*> rows = ps.rows();
    size_t cap = 0;
    for (size_t i = 0; i < nrows; ++i) cap += std::min<size_t>(m, ps.pk[i].exact_len + (mut_off[i + 1] - mut_off[i]));
    uint64_t *d_v, *d_mut;
    const uint8_t* d_flags;
    int rc = upload_list(l, v, m, &d_v);
    if (rc) return rc;
    rc = upload_mut_layers(l, mut_uids, mut_flags, mut_off[nrows], &d_mut, &d_flags);
    if (rc) return rc;
    return ps.synced(csr_to_host(l, cap, nrows, out, out_off, out_cap, [&](uint64_t* d_out, uint64_t* d_off) {
        return list_uids_impl(l, rows.data(), mode, nrows, d_mut, d_flags, mut_off, after_uid, d_v, m, d_out, cap, d_off);
    }));
}

// ---------------------------------------------------------------------------
// List.Uids without a filter, and the count of the same postings, over a task's keys (handleUidPostings)
// ---------------------------------------------------------------------------
// The host-side checks of the four entry points, before anything is copied: the mutable layers, and the bound that
// keeps |S_i| below 2^31.  rows[i] is row i's pack.
template <class Row>
static int list_unfiltered_check(size_t nrows, const uint64_t* mut_off, const void* mut_uids, const void* mut_flags,
                                 const Row* rows) {
    if (int rc = check_mut_layers(mut_off, nrows, mut_uids, mut_flags)) return rc;
    for (size_t r = 0; r < nrows; ++r) {
        const uint64_t n = exact_len(rows[r]) + (mut_off[r + 1] - mut_off[r]);
        if (n >= (uint64_t(1) << 31))
            return fail(DGX_ERR_ARG, "row %zu has %llu postings: at most 2^31 - 1", r, (unsigned long long)n);
    }
    return DGX_OK;
}

// The most values a row keeps for opts.First (posting/list.go:1759-1761, 1841-1843, 1864-1872): 0 is MaxInt32; a
// negative First stops the callback after the first value and the cut keeps it.
static uint64_t first_keep(int32_t first) { return first == 0 ? 0x7fffffffull : first < 0 ? 1 : (uint64_t)first; }

// Rows (d_counts == nullptr) or counts of the unfiltered read (list_uids_unfiltered_kernel.cuh): classify, entry scan,
// rows, and for rows a row scan and the write, so 5 or 3 launches whatever the row count, entry count and pack sizes
// are.  mut_off is host memory, already checked.
static int list_unfiltered_impl(dgx_lane* l, const dgx_dev_pack* const* packs, size_t nrows, const uint64_t* d_mut,
                                const uint8_t* d_flags, const uint64_t* mut_off, uint64_t after, uint64_t first,
                                uint64_t* d_out, size_t out_cap, uint64_t* d_out_off, uint32_t* d_counts) {
    const uint64_t nmut = mut_off[nrows];
    size_t nj = 0;
    for (size_t i = 0; i < nrows; ++i)
        if (packs[i] && packs[i]->pk.nblocks) ++nj;
    if (nj >= kLuuNoJob) return fail(DGX_ERR_ARG, "batch too large for one launch (%zu rows)", nrows);
    // the copied table ends [mut_off | nmut | nrows]
    LuuParams P;
    LuuJob* hj;
    u32* h_rj;
    uint64_t* h_off;
    WsCarve ws(l);
    ws.copied(&P.jobs, &hj, nj);
    ws.copied(&P.row_job, &h_rj, nrows);
    ws.copied(&P.mut_off, &h_off, nrows + 3);
    if (int rc = ws.stage()) return rc;
    uint64_t warps = 0, exact = 0;
    for (size_t i = 0, j = 0; i < nrows; ++i) {
        const dgx_dev_pack* p = packs[i];
        if (!p || p->pk.nblocks == 0) { h_rj[i] = kLuuNoJob; continue; }
        h_rj[i] = (u32)j;
        LuuJob& J = hj[j++];
        J.pk = p->pk;
        J.row = i;
        J.warp_base = warps;
        warps += (p->pk.nblocks + D_BPW - 1) / D_BPW;
        exact += p->exact_len;
    }
    memcpy(h_off, mut_off, (nrows + 1) * sizeof(uint64_t));
    h_off[nrows + 1] = nmut;
    h_off[nrows + 2] = nrows;
    const uint64_t kMaxGrid = 0x7fffffffull;
    const uint64_t g_cls = (nmut + nrows + 255) / 256, g_rows = (nrows + 255) / 256;
    const uint64_t g_write = (warps + D_WARPS - 1) / D_WARPS + (nmut + D_NT - 1) / D_NT;
    const uint64_t t_mut = std::max<uint64_t>((nmut + EN_TILE - 1) / EN_TILE, 1), t_rows = (nrows + EN_TILE - 1) / EN_TILE;
    if (std::max({g_cls, g_write}) > kMaxGrid)
        return fail(DGX_ERR_ARG, "batch too large for one launch (%llu entries, %zu rows)", (unsigned long long)nmut, nrows);
    u64* status;
    u32* tickets;
    ws.zeroed(&status, t_mut + t_rows);
    ws.zeroed(&tickets, 2);
    ws.zeroed(&P.bad, 1);
    ws.plain(&P.cls, nmut);
    ws.plain(&P.cls_ex, nmut + 1);
    ws.plain(&P.rank, nmut);
    ws.plain(&P.skip, nrows);
    ws.plain(&P.sblk, nrows);
    ws.plain(&P.len, nrows);
    if (int rc = ws.commit()) return rc;
    P.njobs = (u32)nj;
    P.nwarps = warps;
    const u64* d_nmut = P.mut_off + nrows + 1;  // scan lengths as device words
    const u64* d_nrows = d_nmut + 1;
    P.nrows = nrows;
    P.mut = (const u64*)d_mut;
    P.flags = d_flags;
    P.nmut = nmut;
    P.after = after;
    P.first = first;
    P.counts = d_counts;
    P.out = (u64*)d_out;
    P.out_cap = out_cap;
    P.out_off = (u64*)d_out_off;
    P.err = l->d_err;
    luu_classify_kernel<<<(unsigned)g_cls, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)t_mut, EN_NT, 0, l->stream>>>(P.cls, P.cls_ex, d_nmut, nmut, status, tickets, nullptr);
    CK(cudaGetLastError());
    luu_rows_kernel<<<(unsigned)g_rows, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    int launches = 3;
    if (!d_counts) {
        scan_u64_kernel<<<(unsigned)t_rows, EN_NT, 0, l->stream>>>(P.len, P.out_off, d_nrows, nrows, status + t_mut,
                                                                    tickets + 1, nullptr);
        CK(cudaGetLastError());
        luu_write_kernel<<<(unsigned)std::max<uint64_t>(g_write, 1), D_NT, sizeof(DWarpSmem) * D_WARPS, l->stream>>>(P);
        CK(cudaGetLastError());
        launches = 5;
    }
    l->launches += launches;
    g_stats.launches += launches;
    g_stats.uids_in += exact + nmut;
    return DGX_OK;
}

extern "C" int dgx_dev_list_uids_unfiltered_rows(dgx_lane* l, const dgx_dev_pack* const* packs, size_t nrows,
                                                 const uint64_t* d_mut_uids, const uint8_t* d_mut_flags,
                                                 const uint64_t* mut_off, uint64_t after_uid, int32_t first,
                                                 uint64_t* d_out, size_t out_cap, uint64_t* d_out_off) {
    if (!l || !d_out_off) return fail(DGX_ERR_ARG, "null argument");
    if (nrows == 0) {
        if (int rc = lane_begin_op(l)) return rc;
        CK(cudaMemsetAsync(d_out_off, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (!packs || !mut_off) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = list_unfiltered_check(nrows, mut_off, d_mut_uids, d_mut_flags, packs)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    const int rc = list_unfiltered_impl(l, packs, nrows, d_mut_uids, d_mut_flags, mut_off, after_uid, first_keep(first),
                                        d_out, out_cap, d_out_off, nullptr);
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    return rc;
}

extern "C" int dgx_dev_list_count_rows(dgx_lane* l, const dgx_dev_pack* const* packs, size_t nrows,
                                       const uint64_t* d_mut_uids, const uint8_t* d_mut_flags, const uint64_t* mut_off,
                                       uint64_t after_uid, uint32_t* d_counts) {
    if (!l) return fail(DGX_ERR_ARG, "null lane");
    if (nrows == 0) return DGX_OK;
    if (!packs || !mut_off || !d_counts) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = list_unfiltered_check(nrows, mut_off, d_mut_uids, d_mut_flags, packs)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    const int rc = list_unfiltered_impl(l, packs, nrows, d_mut_uids, d_mut_flags, mut_off, after_uid, first_keep(0),
                                        nullptr, 0, nullptr, d_counts);
    l->note_output(d_counts, nrows * sizeof(uint32_t));
    return rc;
}

// The host forms: packs staged as in dgx_list_uids_rows, the layers as one copy of uids and one of flags; returns
// the rows (counts == nullptr) or the counts to the host.
static int list_unfiltered_host(const dgx_pack_ref* refs, size_t nrows, const uint64_t* mut_uids,
                                const uint8_t* mut_flags, const uint64_t* mut_off, uint64_t after_uid, int32_t first,
                                uint64_t* out, uint64_t* out_off, size_t out_cap, uint32_t* counts) {
    if (!refs || !mut_off) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = list_unfiltered_check(nrows, mut_off, mut_uids, mut_flags, refs)) return rc;
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    PackSet ps(l, refs, nrows);  // nil / empty packs are packs of no blocks
    if (ps.rc) return ps.rc;
    const uint64_t keep = first_keep(first);
    const std::vector<const dgx_dev_pack*> rows = ps.rows();
    size_t cap = 0;
    for (size_t i = 0; i < nrows; ++i) cap += std::min<uint64_t>(keep, ps.pk[i].exact_len + (mut_off[i + 1] - mut_off[i]));
    uint64_t* d_mut;
    const uint8_t* d_flags;
    int rc = upload_mut_layers(l, mut_uids, mut_flags, mut_off[nrows], &d_mut, &d_flags);
    if (rc) return rc;
    if (counts) {
        void* d_counts;
        rc = l->ws.alloc(nrows * sizeof(uint32_t), &d_counts);
        if (rc) return rc;
        rc = list_unfiltered_impl(l, rows.data(), nrows, d_mut, d_flags, mut_off, after_uid, keep, nullptr, 0, nullptr,
                                  (uint32_t*)d_counts);
        if (rc) return rc;
        CK(cudaMemcpyAsync(counts, d_counts, nrows * sizeof(uint32_t), cudaMemcpyDeviceToHost, l->stream));
        g_stats.d2h += nrows * sizeof(uint32_t);
        return ps.synced(dgx_lane_sync(l));
    }
    return ps.synced(csr_to_host(l, cap, nrows, out, out_off, out_cap, [&](uint64_t* d_out, uint64_t* d_off) {
        return list_unfiltered_impl(l, rows.data(), nrows, d_mut, d_flags, mut_off, after_uid, keep, d_out, cap, d_off,
                                    nullptr);
    }));
}

extern "C" int dgx_list_uids_unfiltered_rows(const dgx_pack_ref* refs, size_t nrows, const uint64_t* mut_uids,
                                             const uint8_t* mut_flags, const uint64_t* mut_off, uint64_t after_uid,
                                             int32_t first, uint64_t* out, uint64_t* out_off, size_t out_cap) {
    if (!out_off) return fail(DGX_ERR_ARG, "null out_off");
    if (nrows == 0) { out_off[0] = 0; return DGX_OK; }
    return list_unfiltered_host(refs, nrows, mut_uids, mut_flags, mut_off, after_uid, first, out, out_off, out_cap,
                                nullptr);
}

extern "C" int dgx_list_count_rows(const dgx_pack_ref* refs, size_t nrows, const uint64_t* mut_uids,
                                   const uint8_t* mut_flags, const uint64_t* mut_off, uint64_t after_uid,
                                   uint32_t* counts) {
    if (nrows == 0) return DGX_OK;
    if (!counts) return fail(DGX_ERR_ARG, "null counts");
    return list_unfiltered_host(refs, nrows, mut_uids, mut_flags, mut_off, after_uid, 0, nullptr, nullptr, 0, counts);
}

// ---------------------------------------------------------------------------
// Backup and restore: codec.DecodeToBuffer / codec.EncodeFromBuffer over a task's keys (backup_codec_kernel.cuh)
// ---------------------------------------------------------------------------
static void count_launches(dgx_lane* l, int n) {
    l->launches += n;
    g_stats.launches += n;
}
// Grid of the grid-stride passes whose length only the device knows (segments, blocks).
static unsigned stride_grid() { return (unsigned)(g_num_sms * 8); }
// Tiles of a scan_u64_kernel over n values, at least one (its grid).
static uint64_t scan_tiles(uint64_t n) { return std::max<uint64_t>(1, (n + EN_TILE - 1) / EN_TILE); }

// Sum of ExactLen over the rows must stay below 2^32: checked before anything is copied.
template <class Row>
static int check_exact_total(const Row* rows, size_t nrows) {
    uint64_t total = 0;
    for (size_t r = 0; r < nrows; ++r) {
        total += exact_len(rows[r]);
        if (total >= (uint64_t(1) << 32))
            return fail(DGX_ERR_ARG, "the packs hold %llu uids or more: at most 2^32 - 1", (unsigned long long)total);
    }
    return DGX_OK;
}

// Packs -> uid_bytes, planned: the job table, the per-block arrays and the look-back words in the lane's workspace.
struct TbRun {
    TbParams P;
    u64* status;
    u32* ticket;
    const u64* d_nblk;
};
static int tb_plan(dgx_lane* l, const dgx_dev_pack* const* packs, size_t nrows, TbRun* R) {
    size_t nj = 0;
    uint64_t nblk = 0, exact = 0;
    for (size_t i = 0; i < nrows; ++i)
        if (packs[i] && packs[i]->pk.nblocks) ++nj;
    // the copied row_blk table ends with nblk again: the scan length as a device word
    TbParams& P = R->P;
    TbJob* hj;
    uint64_t* h_rb;
    WsCarve ws(l);
    ws.copied(&P.jobs, &hj, nj);
    ws.copied(&P.row_blk, &h_rb, nrows + 2);
    if (int rc = ws.stage()) return rc;
    for (size_t i = 0, j = 0; i < nrows; ++i) {
        h_rb[i] = nblk;
        const dgx_dev_pack* p = packs[i];
        if (!p || p->pk.nblocks == 0) continue;
        TbJob& J = hj[j++];
        J.pk = p->pk;
        J.blk0 = nblk;
        J.row = i;
        nblk += p->pk.nblocks;
        exact += p->exact_len;
    }
    h_rb[nrows] = nblk;
    h_rb[nrows + 1] = nblk;
    const size_t tiles = std::max<size_t>(1, (nblk + EN_TILE - 1) / EN_TILE);
    ws.zeroed(&R->status, tiles);
    ws.zeroed(&R->ticket, 4);
    ws.ones(&P.stop, nrows);
    ws.plain(&P.last, nblk);
    ws.plain(&P.bytes, nblk);
    ws.plain(&P.boff, nblk + 1);
    if (int rc = ws.commit()) return rc;
    g_stats.uids_in += exact;
    P.njobs = (u32)nj;
    P.nblk = nblk;
    P.nrows = nrows;
    R->d_nblk = P.row_blk + nrows + 1;
    P.out = nullptr;
    P.out_cap = 0;
    P.out_off = nullptr;
    P.err = nullptr;
    return DGX_OK;
}
// The four launches (blocks, sizes, scan, write); write_only: the write pass again, once the host has sized the output.
static int tb_launch(dgx_lane* l, const TbRun& R, bool write_only) {
    const TbParams& P = R.P;
    const unsigned g_blk = (unsigned)std::max<uint64_t>(1, (P.nblk + 255) / 256);
    int launches = 1;
    if (!write_only) {
        tb_blocks_kernel<<<g_blk, 256, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        tb_sizes_kernel<<<g_blk, 256, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        const unsigned tiles = (unsigned)std::max<uint64_t>(1, (P.nblk + EN_TILE - 1) / EN_TILE);
        scan_u64_kernel<<<tiles, EN_NT, 0, l->stream>>>(P.bytes, P.boff, R.d_nblk, P.nblk, R.status, R.ticket, nullptr);
        CK(cudaGetLastError());
        launches = 4;
    }
    const uint64_t nthreads = std::max<uint64_t>(P.nblk, P.nrows + 1);
    tb_write_kernel<<<(unsigned)((nthreads + 255) / 256), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, launches);
    return DGX_OK;
}

extern "C" int dgx_dev_decode_to_buffer_rows(dgx_lane* l, const dgx_dev_pack* const* packs, size_t nrows, uint8_t* d_out,
                                             size_t out_cap, uint64_t* d_out_off) {
    if (!l || !d_out_off) return fail(DGX_ERR_ARG, "null argument");
    if (nrows == 0) {
        if (int rc = lane_begin_op(l)) return rc;
        CK(cudaMemsetAsync(d_out_off, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (!packs) return fail(DGX_ERR_ARG, "null packs");
    if (int rc = check_exact_total(packs, nrows)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    TbRun R;
    int rc = tb_plan(l, packs, nrows, &R);
    if (rc) return rc;
    R.P.out = d_out;
    R.P.out_cap = out_cap;
    R.P.out_off = (u64*)d_out_off;
    R.P.err = l->d_err;
    rc = tb_launch(l, R, false);
    l->note_output(d_out, out_cap);
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    return rc;
}

extern "C" int dgx_decode_to_buffer_rows(const dgx_pack_ref* refs, size_t nrows, uint8_t* out, uint64_t* out_off,
                                         size_t out_cap) {
    if (!out_off) return fail(DGX_ERR_ARG, "null out_off");
    if (nrows == 0) { out_off[0] = 0; return DGX_OK; }
    if (!refs) return fail(DGX_ERR_ARG, "null refs");
    if (int rc = check_exact_total(refs, nrows)) return rc;
    {  // malformed packs are refused without a device (the staging below walks the same tables again)
        std::vector<uint64_t> uoff;
        for (size_t r = 0; r < nrows; ++r) {
            const dgx_pack_view* v = refs[r].pack;
            if (!v || v->nblocks == 0) continue;
            uoff.resize(v->nblocks + 1);
            uint64_t exact;
            uint32_t max_num;
            if (int rc = walk_block_table(v, uoff.data(), &exact, &max_num)) return rc;
        }
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    PackSet ps(l, refs, nrows);
    if (ps.rc) return ps.rc;
    const std::vector<const dgx_dev_pack*> rows = ps.rows();
    TbRun R;
    int rc = tb_plan(l, rows.data(), nrows, &R);
    if (rc) return rc;
    void* d_off;
    if ((rc = l->ws.alloc((nrows + 1) * sizeof(uint64_t), &d_off))) return rc;
    R.P.out_off = (u64*)d_off;
    if ((rc = tb_launch(l, R, false))) return rc;  // sizes only: the exact byte count is known after this pass
    CK(cudaMemcpyAsync(out_off, d_off, (nrows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if ((rc = dgx_lane_sync(l))) return ps.synced(rc);
    g_stats.d2h += (nrows + 1) * sizeof(uint64_t);
    const uint64_t total = out_off[nrows];
    if (!out || total == 0) return ps.synced(DGX_OK);
    if (total > out_cap)
        return ps.synced(fail(DGX_ERR_CAP, "uid_bytes (%llu bytes) do not fit out_cap (%zu)", (unsigned long long)total, out_cap));
    void* d_out;
    if ((rc = l->ws.alloc(total + 16, &d_out))) return rc;
    R.P.out = (unsigned char*)d_out;
    R.P.out_cap = total;
    if ((rc = tb_launch(l, R, true))) return rc;
    CK(cudaMemcpyAsync(out, d_out, total, cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += total;
    return ps.synced(DGX_OK);
}

// uid_bytes -> packs, planned: the row offsets copied, the look-back words zeroed, the per-value, per-segment and
// per-block arrays in the lane's workspace.  The counts are only known on the device, so the arrays are sized for the
// bound every one of them obeys (values, segments and blocks are at most one per input byte): about 52 bytes per byte.
struct BfRun {
    BfParams P;
    size_t tiles, row_tiles;
    u64 *st_segscan, *st_bytescan, *st_imgscan;
    const u64* d_nrows;
};
static int bf_plan(dgx_lane* l, const uint8_t* d_buf, const uint64_t* buf_off, size_t nrows, uint32_t block_size,
                   BfRun* R) {
    const uint64_t n = buf_off[nrows];
    const size_t T = n / EN_TILE + 1, Tr = nrows / EN_TILE + 1;  // look-back words per scan region
    // the copied row_off table ends with nrows: the scan length as a device word
    BfParams& P = R->P;
    uint64_t* h_off;
    WsCarve ws(l);
    ws.copied(&P.row_off, &h_off, nrows + 2);
    if (int rc = ws.stage()) return rc;
    memcpy(h_off, buf_off, (nrows + 1) * sizeof(uint64_t));
    h_off[nrows + 1] = nrows;
    ws.zeroed(&P.counts, 8);
    ws.zeroed(&P.ticket, 8);
    ws.zeroed(&P.bad, 4);
    ws.zeroed(&P.status, 4 * T + Tr);
    ws.zeroed(&P.sum_flag, T);
    ws.zeroed(&P.sum_val, 2 * T);
    ws.plain(&P.pre, n);
    ws.plain(&P.vrow, n);
    ws.plain(&P.rowbase, nrows);
    ws.plain(&P.seg_start, n + 1);
    ws.plain(&P.seg_cnt, n);
    ws.plain(&P.seg_blk, n + 1);
    ws.plain(&P.blk_bytes, n);
    ws.plain(&P.blk_doff, n + 1);
    ws.plain(&P.brow, n);
    ws.plain(&P.row_blk, nrows + 1);
    ws.plain(&P.img_bytes, nrows);
    if (int rc = ws.commit()) return rc;
    P.buf = d_buf;
    P.n = n;
    R->d_nrows = P.row_off + nrows + 1;
    P.nrows = nrows;
    P.bsz = block_size ? block_size : 1;
    R->st_segscan = P.status + 2 * T;
    R->st_bytescan = P.status + 3 * T;
    R->st_imgscan = P.status + 4 * T;
    R->tiles = (n + EN_TILE - 1) / EN_TILE;
    R->row_tiles = (nrows + EN_TILE - 1) / EN_TILE;
    P.img = nullptr;
    P.img_cap = 0;
    P.img_off = P.nblocks = P.delta_bytes = nullptr;
    P.err = nullptr;
    g_stats.uids_in += n;
    return DGX_OK;
}
// The nine launches; write_only: the write pass again, once the host has sized the images.
static int bf_launch(dgx_lane* l, const BfRun& R, bool write_only) {
    const BfParams& P = R.P;
    const unsigned G = stride_grid(), tiles = (unsigned)R.tiles;
    int launches = 1;
    if (!write_only) {
        bf_values_kernel<<<tiles, EN_NT, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        bf_segments_kernel<<<tiles, EN_NT, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        bf_segcount_kernel<<<G, 256, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        scan_u64_kernel<<<tiles, EN_NT, 0, l->stream>>>(P.seg_cnt, P.seg_blk, P.counts + 1, P.n, R.st_segscan, P.ticket + 2,
                                                         P.counts + 2);
        CK(cudaGetLastError());
        bf_sizes_kernel<<<G, 256, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        scan_u64_kernel<<<tiles, EN_NT, 0, l->stream>>>(P.blk_bytes, P.blk_doff, P.counts + 2, P.n, R.st_bytescan,
                                                         P.ticket + 3, P.counts + 3);
        CK(cudaGetLastError());
        bf_rows_kernel<<<G, 256, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        scan_u64_kernel<<<(unsigned)R.row_tiles, EN_NT, 0, l->stream>>>(P.img_bytes, P.img_off, R.d_nrows, P.nrows,
                                                                         R.st_imgscan, P.ticket + 4, P.counts + 4);
        CK(cudaGetLastError());
        launches = 9;
    }
    bf_write_kernel<<<G, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, launches);
    return DGX_OK;
}
// The checks of both forms before anything is copied; *n gets the byte count.
static int bf_check(const void* buf, const uint64_t* buf_off, size_t nrows, const void* img, const void* nblocks,
                    const void* delta_bytes, uint64_t* n) {
    if (!buf_off || !nblocks || !delta_bytes) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = check_offsets("buf_off", buf_off, nrows, uint64_t(1) << 32)) return rc;
    *n = buf_off[nrows];
    if (*n && !buf) return fail(DGX_ERR_ARG, "null buf");
    if (reinterpret_cast<uintptr_t>(img) & 15u) return fail(DGX_ERR_ARG, "img must be 16-byte aligned");
    return DGX_OK;
}

extern "C" int dgx_dev_encode_from_buffer_rows(dgx_lane* l, const uint8_t* d_buf, const uint64_t* buf_off, size_t nrows,
                                               uint32_t block_size, void* d_img, size_t img_cap, uint64_t* d_img_off,
                                               uint64_t* d_nblocks, uint64_t* d_delta_bytes) {
    if (!l || !d_img_off) return fail(DGX_ERR_ARG, "null argument");
    if (nrows == 0) {
        if (int rc = lane_begin_op(l)) return rc;
        CK(cudaMemsetAsync(d_img_off, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    uint64_t n;
    if (int rc = bf_check(d_buf, buf_off, nrows, d_img, d_nblocks, d_delta_bytes, &n)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_img, img_cap);
    l->note_output(d_img_off, (nrows + 1) * sizeof(uint64_t));
    l->note_output(d_nblocks, nrows * sizeof(uint64_t));
    l->note_output(d_delta_bytes, nrows * sizeof(uint64_t));
    if (n == 0) {  // every row empty: nil packs
        CK(cudaMemsetAsync(d_img_off, 0, (nrows + 1) * sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_nblocks, 0, nrows * sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_delta_bytes, 0, nrows * sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    BfRun R;
    int rc = bf_plan(l, d_buf, buf_off, nrows, block_size, &R);
    if (rc) return rc;
    R.P.img = (unsigned char*)d_img;
    R.P.img_cap = img_cap;
    R.P.img_off = (u64*)d_img_off;
    R.P.nblocks = (u64*)d_nblocks;
    R.P.delta_bytes = (u64*)d_delta_bytes;
    R.P.err = l->d_err;
    return bf_launch(l, R, false);
}

extern "C" int dgx_encode_from_buffer_rows(const uint8_t* buf, const uint64_t* buf_off, size_t nrows, uint32_t block_size,
                                           void* img, size_t img_cap, uint64_t* img_off, uint64_t* nblocks,
                                           uint64_t* delta_bytes) {
    if (!img_off) return fail(DGX_ERR_ARG, "null img_off");
    if (nrows == 0) { img_off[0] = 0; return DGX_OK; }
    uint64_t n;
    if (int rc = bf_check(buf, buf_off, nrows, img, nblocks, delta_bytes, &n)) return rc;
    if (n == 0) {  // every row empty: nil packs
        memset(img_off, 0, (nrows + 1) * sizeof(uint64_t));
        memset(nblocks, 0, nrows * sizeof(uint64_t));
        memset(delta_bytes, 0, nrows * sizeof(uint64_t));
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    void *d_buf, *d_arr;
    int rc = l->ws.alloc(n + 16, &d_buf);
    if (rc) return rc;
    if ((rc = l->ws.alloc((3 * nrows + 1) * sizeof(uint64_t), &d_arr))) return rc;
    CK(cudaMemcpyAsync(d_buf, buf, n, cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += n;
    BfRun R;
    if ((rc = bf_plan(l, (const uint8_t*)d_buf, buf_off, nrows, block_size, &R))) return rc;
    R.P.img_off = (u64*)d_arr;
    R.P.nblocks = R.P.img_off + nrows + 1;
    R.P.delta_bytes = R.P.nblocks + nrows;
    if ((rc = bf_launch(l, R, false))) return rc;  // sizes only: the exact image bytes are known after this pass
    CK(cudaMemcpyAsync(l->h_word, R.P.bad, sizeof(int), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(img_off, R.P.img_off, (nrows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(nblocks, R.P.nblocks, nrows * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(delta_bytes, R.P.delta_bytes, nrows * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if ((rc = dgx_lane_sync(l))) return rc;
    g_stats.d2h += (3 * nrows + 1) * sizeof(uint64_t);
    if (*(const int*)l->h_word) {
        memset(img_off, 0, (nrows + 1) * sizeof(uint64_t));
        memset(nblocks, 0, nrows * sizeof(uint64_t));
        memset(delta_bytes, 0, nrows * sizeof(uint64_t));
        return fail(DGX_ERR_ARG, "a uid_bytes row is not a sequence of valid uvarints");
    }
    const uint64_t total = img_off[nrows];
    if (!img || total == 0) return DGX_OK;
    if (total > img_cap)
        return fail(DGX_ERR_CAP, "pack images (%llu bytes) do not fit img_cap (%zu)", (unsigned long long)total, img_cap);
    void* d_img;
    if ((rc = l->ws.alloc(total, &d_img))) return rc;
    R.P.img = (unsigned char*)d_img;
    R.P.img_cap = total;
    if ((rc = bf_launch(l, R, true))) return rc;
    CK(cudaMemcpyAsync(img, d_img, total, cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += total;
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// MergeSorted over the rows of a uid matrix (sg.DestUIDs = algo.MergeSorted(result.UidMatrix))
// ---------------------------------------------------------------------------
// Sample sort of merge_matrix.cuh: 7 launches plus ceil(log2 ntiles) levels of the sample tree, whatever nrows is.
// Workspace: about 22 bytes per value of v_cap (tile runs 8, keys 4, bucketed values 8, samples, splitters and
// bucket tables about 2.3), plus 24 per chunk of XM_H values.  v_off is read on the device only: no per-row host work.
static int merge_matrix_impl(dgx_lane* l, const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows, uint64_t v_cap,
                             uint64_t* d_out, size_t out_cap, uint64_t* d_out_len) {
    if (nrows == 0 || v_cap == 0) {
        CK(cudaMemsetAsync(d_out_len, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    const uint64_t ntiles = (v_cap + XM_T - 1) / XM_T, ns_cap = ntiles * XM_SPR, nk_cap = 2 * ns_cap + 1;
    const uint64_t nchunks = (v_cap + XM_H - 1) / XM_H;
    const uint64_t t_keys = (nk_cap + EN_TILE - 1) / EN_TILE, t_chunks = (nchunks + EN_TILE - 1) / EN_TILE;
    XmParams P;
    u64 *status, *split, *words;  // words: nsplit, nkeys, nchunks
    u32* tickets;
    WsCarve ws(l);
    ws.zeroed(&P.kcnt, nk_cap);
    ws.zeroed(&P.kfill, nk_cap);
    ws.zeroed(&status, t_keys + t_chunks);
    ws.zeroed(&tickets, 4);
    ws.plain(&P.runs, ntiles * XM_T);
    ws.plain(&P.samples, ns_cap);
    ws.plain(&P.soff, 2 * ntiles);
    ws.plain(&split, ns_cap);
    ws.plain(&words, 4);
    ws.plain(&P.koff, nk_cap + 1);
    ws.plain(&P.bucketed, v_cap);
    ws.plain(&P.cstart, nchunks);
    ws.plain(&P.ccount, nchunks);
    ws.plain(&P.cpos, nchunks + 1);
    ws.plain(&P.rlen, ntiles);
    ws.plain(&P.key, ntiles * XM_T);
    if (int rc = ws.commit()) return rc;
    P.v = (const u64*)d_v;
    P.v_off = (const u64*)d_v_off;
    P.nrows = nrows;
    P.v_cap = v_cap;
    P.split = split;
    P.nsplit = words;
    P.nkeys = words + 1;
    P.nch = words + 2;
    P.ntiles = (u32)ntiles;
    P.nchunks = (u32)nchunks;
    P.out = (u64*)d_out;
    P.out_cap = out_cap;
    P.err = l->d_err;
    xm_tile_kernel<<<(unsigned)ntiles, XM_NT, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    l->launches += 1;
    g_stats.launches += 1;
    // the sample runs are sorted: the merge tree (with de-duplication) yields the distinct splitters
    std::vector<MRef> sruns(ntiles);
    std::vector<uint64_t> sub(ntiles, XM_SPR);
    for (uint64_t t = 0; t < ntiles; ++t) sruns[t] = MRef{P.samples, P.soff + 2 * t, (u64)XM_SPR};
    if (int rc = merge_tree_impl(l, std::move(sruns), std::move(sub), ns_cap, (uint64_t*)split, ns_cap, (uint64_t*)words))
        return rc;
    xm_count_kernel<<<(unsigned)ntiles, XM_NT, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)t_keys, EN_NT, 0, l->stream>>>(P.kcnt, P.koff, P.nkeys, nk_cap, status, tickets, nullptr);
    CK(cudaGetLastError());
    xm_scatter_kernel<<<(unsigned)ntiles, XM_NT, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    xm_chunk_kernel<<<(unsigned)nchunks, XM_CNT, 0, l->stream>>>(P, (u32*)l->d_err + kLaneOverflowWord);
    CK(cudaGetLastError());
    scan_u64_kernel<<<(unsigned)t_chunks, EN_NT, 0, l->stream>>>(P.ccount, P.cpos, P.nch, nchunks, status + t_keys,
                                                                  tickets + 1, (u64*)d_out_len);
    CK(cudaGetLastError());
    xm_gather_kernel<<<(unsigned)nchunks, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    l->launches += 6;
    g_stats.launches += 6;
    return DGX_OK;
}

// Values are counted per 32-bit key and position: 2^32 values or more are refused before anything runs.
constexpr uint64_t kMergeMatrixMax = (uint64_t(1) << 32) - 1;

extern "C" int dgx_dev_merge_sorted_matrix(dgx_lane* l, const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows,
                                           size_t v_cap, uint64_t* d_out, size_t out_cap, uint64_t* d_out_len) {
    if (!l || !d_out_len || (nrows && !d_v_off) || (nrows && v_cap && !d_v)) return fail(DGX_ERR_ARG, "null argument");
    if (v_cap > kMergeMatrixMax) return fail(DGX_ERR_ARG, "v_cap of %zu values: positions are 32-bit", v_cap);
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    const int rc = merge_matrix_impl(l, d_v, d_v_off, nrows, v_cap, d_out, out_cap, d_out_len);
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_out_len, sizeof(uint64_t));
    return rc;
}

extern "C" int dgx_merge_sorted_matrix(const uint64_t* v, const uint64_t* v_off, size_t nrows, uint64_t* out,
                                       size_t out_cap, size_t* out_len) {
    if (nrows == 0) { if (out_len) *out_len = 0; return DGX_OK; }
    if (!v_off) return fail(DGX_ERR_ARG, "null v_off");
    if (int rc = check_offsets("v_off", v_off, nrows, kMergeMatrixMax + 1)) return rc;
    const uint64_t m = v_off[nrows];
    if (m == 0) { if (out_len) *out_len = 0; return DGX_OK; }  // every row empty: nothing runs
    if (!v || (out_cap && !out)) return fail(DGX_ERR_ARG, "null argument");
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += m;
    uint64_t *d_v, *d_off;
    int rc = upload_list(l, v, m, &d_v);  // one copy of the values, one of the offsets
    if (rc) return rc;
    rc = upload_list(l, v_off, nrows + 1, &d_off);
    if (rc) return rc;
    void *d_out, *d_len;
    rc = l->ws.alloc((m + 2) * sizeof(uint64_t), &d_out);
    if (rc) return rc;
    rc = l->ws.alloc(64, &d_len);
    if (rc) return rc;
    rc = merge_matrix_impl(l, d_v, d_off, nrows, m, (uint64_t*)d_out, m, (uint64_t*)d_len);
    if (rc) return rc;
    return finish_to_host(l, (uint64_t*)d_len, (uint64_t*)d_out, m, out, out_cap, out_len);
}

// ---------------------------------------------------------------------------
// @groupby over a uid predicate: a uid matrix inverted into ordered groups per parent row (groupby_kernel.cuh)
// ---------------------------------------------------------------------------
constexpr uint64_t kGbMax = uint64_t(1) << 32;  // rows, parents, dest values, row values and edges are 32-bit counts

static uint32_t gb_bits(uint64_t x) { return x ? 64u - (uint32_t)__builtin_clzll(x) : 0u; }
static unsigned gb_grid(uint64_t n) { return (unsigned)std::max<uint64_t>(1, (n + 255) / 256); }

// The key widths and radix passes of a call, from its sizes alone: parents need b_p = bits(npar - 1), dest ranks
// b_d = bits(ndest - 1), group sizes (at most nrows) b_s = bits(nrows).
struct GbPlan {
    uint32_t b_p, b_d, b_s, p1, p2;
};
static GbPlan gb_plan(uint64_t nrows, uint64_t ndest, uint64_t npar) {
    GbPlan g;
    g.b_p = gb_bits(npar - 1);
    g.b_d = gb_bits(ndest ? ndest - 1 : 0);
    g.b_s = gb_bits(nrows);
    g.p1 = (g.b_p + g.b_d + GB_DIGIT_BITS - 1) / GB_DIGIT_BITS;
    g.p2 = (g.b_p + g.b_s + GB_DIGIT_BITS - 1) / GB_DIGIT_BITS;
    return g;
}

// One stable LSD pass per 8 key bits, ping-ponging between k[0] / p[0] and k[1] / p[1]: the result is in buffer
// passes & 1.  Three launches per pass.  `tiles` radix tiles cover the items; *h_word must hold GB_RADIX * tiles (the
// hist scan's length) and *bad stops every pass.
static int gb_sort(dgx_lane* l, uint64_t tiles, const int* bad, const u64* h_word, u64* const k[2], u32* const p[2],
                   const u64* n_word, uint32_t passes, u64* hist, u64* hoff, u64*& status, u32*& ticket) {
    const uint64_t hn = (uint64_t)GB_RADIX * tiles, ht = (hn + EN_TILE - 1) / EN_TILE;
    for (uint32_t q = 0; q < passes; ++q) {
        const int a = q & 1;
        const u32 shift = q * GB_DIGIT_BITS;
        gb_hist_kernel<<<(unsigned)tiles, GB_NT, 0, l->stream>>>(k[a], n_word, bad, shift, tiles, hist);
        scan_u64_kernel<<<(unsigned)ht, EN_NT, 0, l->stream>>>(hist, hoff, h_word, hn, status, ticket, nullptr);
        gb_scatter_kernel<<<(unsigned)tiles, GB_NT, 0, l->stream>>>(k[a], p[a], n_word, bad, shift, tiles, hoff,
                                                                     k[a ^ 1], p[a ^ 1]);
        CK(cudaGetLastError());
        status += ht;
        ticket += 1;
    }
    count_launches(l, 3 * (int)passes);
    return DGX_OK;
}

// The checks, the pairs and the edge scan: three launches.  Workspace: 24 bytes per parent value of par_cap.
static int gb_front(dgx_lane* l, GbParams& P, u32** tickets) {
    const uint64_t pc = std::max<uint64_t>(P.par_cap, 1), st = (pc + EN_TILE - 1) / EN_TILE;
    // the words are zeroed, so a refused input leaves every count at 0
    u64* status;
    WsCarve ws(l);
    ws.zeroed(&P.bad, 16);
    ws.zeroed(&P.words, GB_WORDS);
    ws.zeroed(tickets, 32);
    ws.zeroed(&status, st);
    ws.plain(&P.plen, pc);
    ws.plain(&P.eoff, pc + 1);
    ws.plain(&P.prow, pc);
    ws.plain(&P.ppar, pc);
    if (int rc = ws.commit()) return rc;
    P.err = l->d_err;
    const uint64_t nt = std::max(std::max(P.nrows + 1, P.npar + 1), std::max(P.ndest, P.v_cap));
    gb_check_kernel<<<gb_grid(nt), 256, 0, l->stream>>>(P);
    gb_pairs_kernel<<<gb_grid(pc), 256, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)st, EN_NT, 0, l->stream>>>(P.plen, P.eoff, P.words + GB_W_PV, P.par_cap, status,
                                                           *tickets, P.words + GB_W_E);
    CK(cudaGetLastError());
    count_launches(l, 3);
    *tickets += 1;
    return DGX_OK;
}

// Expand, both sorts, the groups and the write: 8 + 3 (P1 + P2) launches.  Workspace: 94 bytes per edge of e_cap
// (edge keys and rows twice 24, heads and group indices 16, group starts, order keys twice and group of each position
// 36, sizes and offsets 16, positions 4, hist and its scan 2).
static int gb_back(dgx_lane* l, GbParams& P, const GbPlan& g, u32* ticket) {
    const uint64_t ec = std::max<uint64_t>(P.e_cap, 1);
    P.tiles = (ec + GB_TILE - 1) / GB_TILE;
    const uint64_t hn = (uint64_t)GB_RADIX * P.tiles, ht = (hn + EN_TILE - 1) / EN_TILE, et = (ec + EN_TILE - 1) / EN_TILE;
    u64 *status, *ek[2], *gk[2], *hist, *hoff;
    u32 *ep[2], *gp[2];
    WsCarve ws(l);
    ws.zeroed(&status, (g.p1 + g.p2) * ht + 2 * et);
    ws.plain(&ek[0], ec);
    ws.plain(&ek[1], ec);
    ws.plain(&P.head, ec);
    ws.plain(&P.gidx, ec + 1);
    ws.plain(&P.gstart, ec + 1);
    ws.plain(&gk[0], ec);
    ws.plain(&gk[1], ec);
    ws.plain(&P.gsz, ec);
    ws.plain(&P.moff, ec + 1);
    ws.plain(&hist, hn);
    ws.plain(&hoff, hn + 1);
    ws.plain(&ep[0], ec);
    ws.plain(&ep[1], ec);
    ws.plain(&gp[0], ec);
    ws.plain(&gp[1], ec);
    ws.plain(&P.inv, ec);
    if (int rc = ws.commit()) return rc;
    P.ek = ek[0];
    P.ep = ep[0];
    gb_expand_kernel<<<gb_grid(ec), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    if (int rc = gb_sort(l, P.tiles, P.bad, P.words + GB_W_H, ek, ep, P.words + GB_W_E, g.p1, hist, hoff, status,
                         ticket))
        return rc;
    P.ek = ek[g.p1 & 1];
    P.ep = ep[g.p1 & 1];
    gb_heads_kernel<<<gb_grid(ec), 256, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)et, EN_NT, 0, l->stream>>>(P.head, P.gidx, P.words + GB_W_E, P.e_cap, status, ticket,
                                                           P.words + GB_W_G);
    status += et;
    ticket += 1;
    gb_groups_kernel<<<gb_grid(ec), 256, 0, l->stream>>>(P);
    gb_gkeys_kernel<<<gb_grid(ec), 256, 0, l->stream>>>(P, gk[0], gp[0]);
    CK(cudaGetLastError());
    if (int rc = gb_sort(l, P.tiles, P.bad, P.words + GB_W_H, gk, gp, P.words + GB_W_G, g.p2, hist, hoff, status,
                         ticket))
        return rc;
    P.gk = gk[g.p2 & 1];
    P.gp = gp[g.p2 & 1];
    gb_sizes_kernel<<<gb_grid(ec), 256, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)et, EN_NT, 0, l->stream>>>(P.gsz, P.moff, P.words + GB_W_G, P.e_cap, status, ticket,
                                                           nullptr);
    gb_write_kernel<<<gb_grid(std::max<uint64_t>(ec + 1, P.npar + 1)), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 8);
    return DGX_OK;
}

static GbParams gb_params(const uint64_t* src, size_t nrows, const uint64_t* v, const uint64_t* v_off, uint64_t v_cap,
                          const uint64_t* dest, size_t ndest, const uint64_t* par, const uint64_t* par_off, size_t npar,
                          uint64_t par_cap, const GbPlan& g) {
    GbParams P{};
    P.src = (const u64*)src;
    P.nrows = nrows;
    P.v = (const u64*)v;
    P.v_off = (const u64*)v_off;
    P.v_cap = v_cap;
    P.dest = (const u64*)dest;
    P.ndest = ndest;
    P.par = (const u64*)par;
    P.par_off = (const u64*)par_off;
    P.npar = npar;
    P.par_cap = par_cap;
    P.b_d = g.b_d;
    P.b_s = g.b_s;
    return P;
}

extern "C" int dgx_dev_groupby_uid(dgx_lane* l, const uint64_t* d_src, size_t nrows, const uint64_t* d_v,
                                   const uint64_t* d_v_off, size_t v_cap, const uint64_t* d_dest, size_t ndest,
                                   const uint64_t* d_par, const uint64_t* d_par_off, size_t npar, size_t par_cap,
                                   size_t e_cap, uint64_t* d_keys, uint64_t* d_grp_off, uint64_t* d_mem_off,
                                   size_t grp_cap, uint64_t* d_members, size_t mem_cap, uint64_t* d_sizes) {
    if (!l || !d_sizes || !d_grp_off || !d_mem_off) return fail(DGX_ERR_ARG, "null argument");
    if (nrows >= kGbMax || npar >= kGbMax || ndest >= kGbMax || v_cap >= kGbMax || par_cap >= kGbMax || e_cap >= kGbMax)
        return fail(DGX_ERR_ARG, "groupby sizes are 32-bit: nrows, npar, ndest, v_cap, par_cap and e_cap below 2^32");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_grp_off, (npar + 1) * sizeof(uint64_t));
    l->note_output(d_mem_off, (grp_cap + 1) * sizeof(uint64_t));
    l->note_output(d_sizes, 2 * sizeof(uint64_t));
    if (npar == 0 || nrows == 0 || v_cap == 0 || par_cap == 0) {  // no edge can exist: zero groups
        CK(cudaMemsetAsync(d_grp_off, 0, (npar + 1) * sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_mem_off, 0, sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_sizes, 0, 2 * sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (!d_src || !d_v || !d_v_off || !d_par || !d_par_off || (ndest && !d_dest) || (grp_cap && !d_keys))
        return fail(DGX_ERR_ARG, "null argument");
    const GbPlan g = gb_plan(nrows, ndest, npar);
    GbParams P = gb_params(d_src, nrows, d_v, d_v_off, v_cap, d_dest, ndest, d_par, d_par_off, npar, par_cap, g);
    P.e_cap = e_cap;
    P.keys = (u64*)d_keys;
    P.grp_off = (u64*)d_grp_off;
    P.mem_off = (u64*)d_mem_off;
    P.members = (u64*)d_members;
    P.grp_cap = grp_cap;
    P.mem_cap = mem_cap;
    P.sizes = (u64*)d_sizes;
    u32* tickets;
    if (int rc = gb_front(l, P, &tickets)) return rc;
    if (int rc = gb_back(l, P, g, tickets)) return rc;
    l->note_output(d_keys, grp_cap * sizeof(uint64_t));
    l->note_output(d_members, mem_cap * sizeof(uint64_t));
    return DGX_OK;
}

extern "C" int dgx_groupby_uid(const uint64_t* src, size_t nrows, const uint64_t* v, const uint64_t* v_off,
                               const uint64_t* dest, size_t ndest, const uint64_t* par, const uint64_t* par_off,
                               size_t npar, uint64_t* keys, uint64_t* grp_off, uint64_t* mem_off, size_t grp_cap,
                               uint64_t* members, size_t mem_cap, size_t* ngroups, size_t* nmembers) {
    if (!ngroups || !nmembers || !grp_off || !mem_off || (npar && !par_off) || (nrows && !v_off))
        return fail(DGX_ERR_ARG, "null argument");
    if (nrows >= kGbMax || npar >= kGbMax || ndest >= kGbMax)
        return fail(DGX_ERR_ARG, "groupby sizes are 32-bit: nrows, npar and ndest below 2^32");
    if (nrows) if (int rc = check_offsets("v_off", v_off, nrows, kGbMax)) return rc;
    if (npar) if (int rc = check_offsets("par_off", par_off, npar, kGbMax)) return rc;
    const uint64_t m = nrows ? v_off[nrows] : 0, pv = npar ? par_off[npar] : 0;
    auto none = [&]() {  // zero groups: every parent owns none
        memset(grp_off, 0, (npar + 1) * sizeof(uint64_t));
        mem_off[0] = 0;
        *ngroups = *nmembers = 0;
        return DGX_OK;
    };
    if (m == 0 || pv == 0) return none();
    if (!src || !v || !par || (ndest && !dest) || (grp_cap && !keys)) return fail(DGX_ERR_ARG, "null argument");
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += nrows + m + ndest + pv;
    uint64_t *d_src, *d_v, *d_v_off, *d_dest, *d_par, *d_par_off;  // one copy each
    int rc;
    if ((rc = upload_list(l, src, nrows, &d_src)) || (rc = upload_list(l, v, m, &d_v)) ||
        (rc = upload_list(l, v_off, nrows + 1, &d_v_off)) || (rc = upload_list(l, dest, ndest, &d_dest)) ||
        (rc = upload_list(l, par, pv, &d_par)) || (rc = upload_list(l, par_off, npar + 1, &d_par_off)))
        return rc;
    const GbPlan g = gb_plan(nrows, ndest, npar);
    GbParams P = gb_params(d_src, nrows, d_v, d_v_off, m, d_dest, ndest, d_par, d_par_off, npar, pv, g);
    u32* tickets;
    if ((rc = gb_front(l, P, &tickets))) return rc;
    // the edge count sizes the rest: one round trip, which also surfaces a refused input
    CK(cudaMemcpyAsync(l->h_word, P.words + GB_W_E, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if ((rc = dgx_lane_sync(l))) return rc;
    const uint64_t E = l->h_word[0];
    if (E == 0) return none();
    if (E >= kGbMax) return fail(DGX_ERR_ARG, "%llu restricted edges: at most 2^32 - 1", (unsigned long long)E);
    u64* d_members;
    WsCarve o(l);
    o.plain(&P.keys, E);
    o.plain(&d_members, E);
    o.plain(&P.mem_off, E + 1);
    o.plain(&P.grp_off, npar + 1);
    o.plain(&P.sizes, 2);
    if ((rc = o.commit())) return rc;
    P.members = members ? d_members : nullptr;
    P.e_cap = P.grp_cap = P.mem_cap = E;
    if ((rc = gb_back(l, P, g, tickets))) return rc;
    CK(cudaMemcpyAsync(l->h_word, P.sizes, 2 * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if ((rc = dgx_lane_sync(l))) return rc;
    const uint64_t G = l->h_word[0];
    *ngroups = G;
    *nmembers = E;
    if (G > grp_cap || (members && E > mem_cap))
        return fail(DGX_ERR_CAP, "%llu groups of %llu members do not fit grp_cap %zu / mem_cap %zu",
                    (unsigned long long)G, (unsigned long long)E, grp_cap, mem_cap);
    if (G) CK(cudaMemcpyAsync(keys, P.keys, G * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(mem_off, P.mem_off, (G + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(grp_off, P.grp_off, (npar + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (members) CK(cudaMemcpyAsync(members, P.members, E * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += (2 * G + npar + 2 + (members ? E : 0)) * sizeof(uint64_t);
    g_stats.uids_out += members ? E : G;
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// @recurse: each sg's uid matrix filtered against the edges already taken, in HBM (recurse_kernel.cuh)
// ---------------------------------------------------------------------------
constexpr uint64_t kRcMax = uint64_t(1) << 32;  // rows, values and set sizes are 32-bit counts

// Buffer b holds from[] at buf[b] and to[] at buf[b] + cap.  Which buffer is current, and the size, are device words
// (d_state) that queued steps update; size / cur mirror them as of the last wait, and bound is the size then plus the
// v_cap of every step queued since, which sizes the capacity without a round trip.
struct dgx_reach_set {
    std::mutex mu;
    int device = 0;
    uint64_t* buf[2] = {nullptr, nullptr};
    uint64_t cap = 0;
    uint64_t* d_state = nullptr;  // [current buffer, size]
    uint64_t size = 0, cur = 0, bound = 0;
    dgx_lane* lane = nullptr;     // the lane of the device-form steps queued since the last wait
    std::vector<void*> retired;   // buffers replaced by growth, still read by queued steps until the next wait
};

static void rc_free_retired(dgx_reach_set* s) {
    for (void* p : s->retired) cudaFree(p);
    s->retired.clear();
}

// Waits for the set's queued steps and reads its words back.  Caller holds s->mu.
static int rc_wait(dgx_reach_set* s) {
    CK(cudaSetDevice(s->device));
    if (!s->lane) return DGX_OK;
    uint64_t st[2];
    CK(cudaMemcpyAsync(st, s->d_state, sizeof(st), cudaMemcpyDeviceToHost, s->lane->stream));
    CK(cudaStreamSynchronize(s->lane->stream));
    s->cur = st[0];
    s->size = s->bound = st[1];
    s->lane = nullptr;
    rc_free_retired(s);
    return DGX_OK;
}

// Capacity for `need` edges: both buffers grow geometrically, their first `bound` records copied on the stream (the
// current buffer is only known on the device).  The new buffers replace the old ones only once every copy is queued,
// so an allocation or a copy that fails leaves the set as it was.
static int rc_reserve(dgx_reach_set* s, cudaStream_t stream, uint64_t need) {
    if (need <= s->cap) return DGX_OK;
    const uint64_t ncap = std::max(need, 2 * s->cap);
    uint64_t* nb[2] = {nullptr, nullptr};
    auto drop = [&](int code, const char* what) {
        cudaGetLastError();
        for (uint64_t* p : nb) if (p) cudaFree(p);
        return fail(code, "reach set growth to %llu edges: %s failed", (unsigned long long)ncap, what);
    };
    for (int b = 0; b < 2; ++b)
        if (cudaMalloc(&nb[b], 2 * ncap * sizeof(uint64_t)) != cudaSuccess) return drop(DGX_ERR_OOM, "cudaMalloc");
    for (int b = 0; b < 2; ++b)
        if (s->bound && (s->lane || (uint64_t)b == s->cur)) {  // an idle set's other buffer holds nothing live
            const size_t bytes = s->bound * sizeof(uint64_t);
            if (cudaMemcpyAsync(nb[b], s->buf[b], bytes, cudaMemcpyDeviceToDevice, stream) != cudaSuccess ||
                cudaMemcpyAsync(nb[b] + ncap, s->buf[b] + s->cap, bytes, cudaMemcpyDeviceToDevice, stream) != cudaSuccess) {
                if (stream) cudaStreamSynchronize(stream);  // copies already queued read and write nb
                return drop(DGX_ERR_CUDA, "cudaMemcpyAsync");
            }
        }
    for (int b = 0; b < 2; ++b) {
        if (s->buf[b]) s->retired.push_back(s->buf[b]);
        s->buf[b] = nb[b];
    }
    s->cap = ncap;
    return DGX_OK;
}

extern "C" int dgx_reach_create(const uint64_t* from, const uint64_t* to, size_t n, dgx_reach_set** set) {
    if (!set || (n && (!from || !to))) return fail(DGX_ERR_ARG, "null argument");
    if (n >= kRcMax) return fail(DGX_ERR_ARG, "%zu edges: a reach set holds at most 2^32 - 1", n);
    for (size_t k = 1; k < n; ++k)
        if (from[k - 1] > from[k] || (from[k - 1] == from[k] && to[k - 1] >= to[k]))
            return fail(DGX_ERR_ARG, "edge %zu does not strictly ascend by (from, to)", k);
    if (int rc = dgx_init(-1)) return rc;
    CK(cudaSetDevice(g_device));
    dgx_reach_set* s = new dgx_reach_set();
    s->device = g_device;
    int rc = DGX_OK;
    if (cudaMalloc(&s->d_state, 2 * sizeof(uint64_t)) != cudaSuccess) rc = fail(DGX_ERR_OOM, "reach set allocation failed");
    if (!rc) rc = rc_reserve(s, nullptr, std::max<uint64_t>(n, 1024));
    const uint64_t st[2] = {0, n};
    if (!rc && n &&
        (cudaMemcpy(s->buf[0], from, n * sizeof(uint64_t), cudaMemcpyHostToDevice) != cudaSuccess ||
         cudaMemcpy(s->buf[0] + s->cap, to, n * sizeof(uint64_t), cudaMemcpyHostToDevice) != cudaSuccess))
        rc = fail(DGX_ERR_CUDA, "reach set upload failed");
    if (!rc && cudaMemcpy(s->d_state, st, sizeof(st), cudaMemcpyHostToDevice) != cudaSuccess)
        rc = fail(DGX_ERR_CUDA, "reach set upload failed");
    rc_free_retired(s);
    s->size = s->bound = n;
    if (rc) {
        dgx_reach_destroy(s);
        return rc;
    }
    g_stats.h2d += 2 * n * sizeof(uint64_t);
    *set = s;
    return DGX_OK;
}

extern "C" void dgx_reach_destroy(dgx_reach_set* s) {
    if (!s) return;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        rc_wait(s);
        rc_free_retired(s);
        for (uint64_t* b : s->buf) if (b) cudaFree(b);
        if (s->d_state) cudaFree(s->d_state);
    }
    delete s;
}

extern "C" int dgx_reach_size(dgx_reach_set* s, size_t* n) {
    if (!s || !n) return fail(DGX_ERR_ARG, "null argument");
    std::lock_guard<std::mutex> lk(s->mu);
    if (int rc = rc_wait(s)) return rc;
    *n = s->size;
    return DGX_OK;
}

extern "C" int dgx_reach_export(dgx_reach_set* s, uint64_t* from, uint64_t* to, size_t cap, size_t* n) {
    if (!s || !n) return fail(DGX_ERR_ARG, "null argument");
    std::lock_guard<std::mutex> lk(s->mu);
    if (int rc = rc_wait(s)) return rc;
    *n = s->size;
    if (s->size > cap) return fail(DGX_ERR_CAP, "%llu edges do not fit cap %zu", (unsigned long long)s->size, cap);
    if (s->size && (!from || !to)) return fail(DGX_ERR_ARG, "null argument");
    if (s->size) {
        CK(cudaMemcpy(from, s->buf[s->cur], s->size * sizeof(uint64_t), cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(to, s->buf[s->cur] + s->cap, s->size * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    }
    g_stats.d2h += 2 * s->size * sizeof(uint64_t);
    return DGX_OK;
}

// One step on the lane, for a set with room for bound + v_cap edges: 5 launches, the matrix merge's, 2 launches.
// Workspace: 28 bytes per value of v_cap (row 4, keep flag 8, its scan 8, kept from 8), 24 per row (slice bounds 16,
// the merge's offsets 8), the merge's about 22 per value, and the scan's look-back words.  d_out_off and d_sizes are
// written by the kernels.
static int rc_step(dgx_lane* l, dgx_reach_set* s, const uint64_t* d_src, size_t nrows, const uint64_t* d_v,
                   const uint64_t* d_v_off, uint64_t v_cap, const uint64_t* d_dest, size_t ndest, uint64_t* d_out,
                   uint64_t* d_out_off, uint64_t* d_dest_out, size_t dest_cap, uint64_t* d_sizes) {
    const uint64_t tiles = (v_cap + EN_TILE - 1) / EN_TILE;
    RcParams P;
    u64* status;
    u32* ticket;
    WsCarve ws(l);
    ws.zeroed(&P.bad, 4);
    ws.zeroed(&P.words, RC_WORDS);
    ws.zeroed(&ticket, 6);
    ws.zeroed(&status, tiles);
    ws.plain(&P.lo, nrows);
    ws.plain(&P.hi, nrows);
    ws.plain(&P.w_off, nrows + 1);
    ws.plain(&P.keep, v_cap);
    ws.plain(&P.kex, v_cap + 1);
    ws.plain(&P.kfrom, v_cap);
    ws.plain(&P.row, v_cap);
    if (int rc = ws.commit()) return rc;
    P.src = (const u64*)d_src;
    P.nrows = nrows;
    P.v = (const u64*)d_v;
    P.v_off = (const u64*)d_v_off;
    P.v_cap = v_cap;
    P.dest = (const u64*)d_dest;
    P.ndest = d_dest ? ndest : 0;
    for (int b = 0; b < 2; ++b) {
        P.sfrom[b] = (u64*)s->buf[b];
        P.sto[b] = (u64*)s->buf[b] + s->cap;
    }
    P.state = (u64*)s->d_state;
    P.out = (u64*)d_out;
    P.out_off = (u64*)d_out_off;
    P.sizes = (u64*)d_sizes;
    P.err = l->d_err;
    const uint64_t nt = std::max<uint64_t>(std::max<uint64_t>(nrows + 1, v_cap), P.ndest);
    rc_check_kernel<<<gb_grid(nt), 256, 0, l->stream>>>(P);
    rc_locate_kernel<<<gb_grid(nrows), 256, 0, l->stream>>>(P);
    rc_flags_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)tiles, EN_NT, 0, l->stream>>>(P.keep, P.kex, P.words + RC_W_M, v_cap, status, ticket,
                                                                P.words + RC_W_K);
    rc_gather_kernel<<<gb_grid(std::max<uint64_t>(v_cap, nrows + 1)), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 5);
    if (int rc = merge_matrix_impl(l, d_out, (const uint64_t*)P.w_off, nrows, v_cap, d_dest_out, dest_cap,
                                   (uint64_t*)(P.words + RC_W_D)))
        return rc;
    rc_insert_kernel<<<stride_grid(), 256, 0, l->stream>>>(P);
    rc_commit_kernel<<<1, 1, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 2);
    return DGX_OK;
}

// The checks both forms make before anything is copied.  Caller holds s->mu.
static int rc_check_step(dgx_reach_set* s, const dgx_lane* l, size_t nrows, uint64_t m, size_t out_cap,
                         size_t dest_cap) {
    if (s->lane && s->lane != l)
        return fail(DGX_ERR_ARG, "the reach set has steps queued on another lane: wait for them with dgx_reach_size");
    if (nrows >= kRcMax || m >= kRcMax) return fail(DGX_ERR_ARG, "recurse sizes are 32-bit: nrows and values below 2^32");
    if (s->bound + m >= kRcMax)
        return fail(DGX_ERR_ARG, "the reach set could reach %llu edges: at most 2^32 - 1",
                    (unsigned long long)(s->bound + m));
    if (out_cap < m || dest_cap < m)
        return fail(DGX_ERR_CAP, "out_cap %zu / dest_cap %zu below the %llu values", out_cap, dest_cap,
                    (unsigned long long)m);
    return DGX_OK;
}

extern "C" int dgx_dev_recurse_filter(dgx_lane* l, dgx_reach_set* s, const uint64_t* d_src, size_t nrows,
                                      const uint64_t* d_v, const uint64_t* d_v_off, size_t v_cap,
                                      const uint64_t* d_dest, size_t ndest, uint64_t* d_out, uint64_t* d_out_off,
                                      size_t out_cap, uint64_t* d_dest_out, size_t dest_cap, uint64_t* d_sizes) {
    if (!l || !s || !d_sizes || !d_out_off) return fail(DGX_ERR_ARG, "null argument");
    if (nrows && v_cap && (!d_src || !d_v || !d_v_off || !d_out || !d_dest_out))
        return fail(DGX_ERR_ARG, "null argument");
    if (d_dest && ndest >= kRcMax) return fail(DGX_ERR_ARG, "ndest of %zu: at most 2^32 - 1", ndest);
    std::lock_guard<std::mutex> lk(s->mu);
    if (int rc = rc_check_step(s, l, nrows, v_cap, out_cap, dest_cap)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    l->note_output(d_sizes, 2 * sizeof(uint64_t));
    if (nrows == 0 || v_cap == 0) {  // no edge: nothing is kept
        CK(cudaMemsetAsync(d_out_off, 0, (nrows + 1) * sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_sizes, 0, 2 * sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (int rc = rc_reserve(s, l->stream, s->bound + v_cap)) return rc;
    s->lane = l;  // queued copies or steps now read the set
    s->bound += v_cap;
    if (int rc = rc_step(l, s, d_src, nrows, d_v, d_v_off, v_cap, d_dest, ndest, d_out, d_out_off, d_dest_out,
                         dest_cap, d_sizes))
        return rc;
    g_stats.uids_in += v_cap;
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_dest_out, dest_cap * sizeof(uint64_t));
    return DGX_OK;
}

extern "C" int dgx_recurse_filter(dgx_reach_set* s, const uint64_t* src, size_t nrows, const uint64_t* v,
                                  const uint64_t* v_off, const uint64_t* dest, size_t ndest, uint64_t* out,
                                  uint64_t* out_off, size_t out_cap, uint64_t* dest_out, size_t dest_cap,
                                  size_t* dest_len) {
    if (!s || !out_off || !dest_len || (nrows && !v_off)) return fail(DGX_ERR_ARG, "null argument");
    if (nrows >= kRcMax) return fail(DGX_ERR_ARG, "recurse sizes are 32-bit: nrows below 2^32");
    if (nrows) if (int rc = check_offsets("v_off", v_off, nrows, kRcMax)) return rc;
    const uint64_t m = nrows ? v_off[nrows] : 0;
    if (m && (!src || !v || !out || !dest_out)) return fail(DGX_ERR_ARG, "null argument");
    if (dest && ndest >= kRcMax) return fail(DGX_ERR_ARG, "ndest of %zu: at most 2^32 - 1", ndest);
    std::lock_guard<std::mutex> lk(s->mu);
    if (int rc = rc_check_step(s, nullptr, nrows, m, out_cap, dest_cap)) return rc;
    if (m == 0) {
        memset(out_off, 0, (nrows + 1) * sizeof(uint64_t));
        *dest_len = 0;
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += nrows + m + (dest ? ndest : 0);
    uint64_t *d_src, *d_v, *d_v_off, *d_dest = nullptr;
    int rc;
    if ((rc = upload_list(l, src, nrows, &d_src)) || (rc = upload_list(l, v, m, &d_v)) ||
        (rc = upload_list(l, v_off, nrows + 1, &d_v_off)) || (dest && (rc = upload_list(l, dest, ndest, &d_dest))))
        return rc;
    uint64_t *d_sizes, *d_out, *d_dest_out, *d_off;
    WsCarve o(l);
    o.plain(&d_sizes, 2);
    o.plain(&d_out, m);
    o.plain(&d_dest_out, m);
    o.plain(&d_off, nrows + 1);
    if ((rc = o.commit())) return rc;
    if ((rc = rc_reserve(s, l->stream, s->bound + m))) return rc;
    s->lane = l;  // waited for below, whatever happens
    s->bound += m;
    rc = rc_step(l, s, d_src, nrows, d_v, d_v_off, m, d_dest, ndest, d_out, d_off, d_dest_out, m, d_sizes);
    if (!rc) CK(cudaMemcpyAsync(l->h_word, d_sizes, 2 * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (int wrc = rc_wait(s)) return wrc;
    if (rc || (rc = dgx_lane_sync(l))) return rc;
    const uint64_t K = l->h_word[0], D = l->h_word[1];
    CK(cudaMemcpyAsync(out_off, d_off, (nrows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (K) CK(cudaMemcpyAsync(out, d_out, K * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (D) CK(cudaMemcpyAsync(dest_out, d_dest_out, D * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    *dest_len = D;
    g_stats.d2h += (K + D + nrows + 3) * sizeof(uint64_t);
    g_stats.uids_out += K + D;
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// @cascade: a forest's uid matrices pruned bottom-up, with cascade pagination, in one call (cascade_kernel.cuh)
// ---------------------------------------------------------------------------
constexpr size_t kCcMaxNodes = size_t(1) << 16;
constexpr uint32_t kCcMaxDepth = 64;            // levels: a node's depth is at most kCcMaxDepth - 1
constexpr uint64_t kCcMax = uint64_t(1) << 32;  // rows, values and dest values in all are 32-bit counts

// One node's arrays, node order: host pointers (host form) or device pointers, which only the kernels read.
struct CcSrc {
    const uint64_t* v;
    const uint64_t* v_off;
    uint64_t v_base, nrows, vcap;
    const uint64_t* dest;
    uint64_t ndest;
    const uint8_t* hv;
    uint64_t nhv;
};

struct CcPlan {
    std::vector<CcNode> node;    // level order
    std::vector<uint32_t> ck;    // checked children, level-order indices
    std::vector<CcLevel> level;  // the levels with work, deepest first
    uint64_t nv = 0, no = 0, nd = 0, nh = 0, rows = 0, max_nv = 0, max_nd = 0;
};

static int cc_check_tree(const dgx_cascade_tree* t) {
    if (!t) return fail(DGX_ERR_ARG, "null tree");
    const size_t n = t->nnodes;
    if (n >= kCcMaxNodes) return fail(DGX_ERR_ARG, "%zu nodes: at most 2^16 - 1", n);
    if (n && (!t->parent || !t->flags || !t->first || !t->offset || !t->counts_len))
        return fail(DGX_ERR_ARG, "null tree array");
    std::vector<uint32_t> depth(n);
    for (size_t k = 0; k < n; ++k) {
        const uint32_t p = t->parent[k];
        if (t->flags[k] & ~uint8_t(DGX_CASCADE_CASCADE | DGX_CASCADE_CHECKED | DGX_CASCADE_FILTERED |
                                   DGX_CASCADE_ORDERED | DGX_CASCADE_SKIP))
            return fail(DGX_ERR_ARG, "node %zu: unknown flag bits 0x%x", k, (unsigned)t->flags[k]);
        if (p == UINT32_MAX) { depth[k] = 0; continue; }
        if (p >= k) return fail(DGX_ERR_ARG, "node %zu: parent %u is not below it", k, p);
        if (t->flags[p] & DGX_CASCADE_SKIP) return fail(DGX_ERR_ARG, "node %zu: its parent %u is SKIP", k, p);
        depth[k] = depth[p] + 1;
        if (depth[k] >= kCcMaxDepth) return fail(DGX_ERR_ARG, "node %zu is deeper than %u", k, kCcMaxDepth - 1);
    }
    return DGX_OK;
}

// The level-order plan of a checked tree: modes, slots, checked children and the levels with work.
static void cc_plan(const dgx_cascade_tree* t, const CcSrc* src, CcPlan* P) {
    const size_t n = t->nnodes;
    std::vector<uint32_t> depth(n), pos(n);
    uint32_t maxd = 0;
    for (size_t k = 0; k < n; ++k) {
        depth[k] = t->parent[k] == UINT32_MAX ? 0 : depth[t->parent[k]] + 1;
        maxd = std::max(maxd, depth[k]);
    }
    std::vector<uint32_t> order;  // deepest level first, node order inside a level
    std::vector<uint32_t> lb;     // level boundaries in `order`
    for (int64_t d = maxd; d >= 0 && n; --d) {
        lb.push_back((uint32_t)order.size());
        for (size_t k = 0; k < n; ++k)
            if (depth[k] == (uint32_t)d) { pos[k] = (uint32_t)order.size(); order.push_back((uint32_t)k); }
    }
    lb.push_back((uint32_t)order.size());
    std::vector<uint64_t> out_row(n + 1, 0);
    for (size_t k = 0; k < n; ++k) out_row[k + 1] = out_row[k] + src[k].nrows;
    P->rows = out_row[n];
    std::vector<std::vector<uint32_t>> checked(n);
    for (size_t k = 0; k < n; ++k)
        if (t->parent[k] != UINT32_MAX && (t->flags[k] & DGX_CASCADE_CHECKED)) checked[t->parent[k]].push_back(pos[k]);
    P->node.resize(n);
    for (size_t q = 0; q < n; ++q) {
        const uint32_t k = order[q];
        const CcSrc& s = src[k];
        const uint8_t f = t->flags[k];
        const bool root = t->parent[k] == UINT32_MAX, cascade = f & DGX_CASCADE_CASCADE, skip = f & DGX_CASCADE_SKIP;
        CcNode& c = P->node[q];
        c.v = (const u64*)s.v;
        c.v_off = (const u64*)s.v_off;
        c.dest = (const u64*)s.dest;
        c.hv = s.hv;
        c.v_base = s.v_base;
        c.vb = P->nv;
        c.vcap = s.vcap;
        c.ob = P->no;
        c.nrows = s.nrows;
        c.db = P->nd;
        c.ndest = s.ndest;
        c.hb = P->nh;
        c.nhv = s.nhv;
        c.counts_len = t->counts_len[k];
        c.out_row = out_row[k];
        c.id = k;
        const bool paged = cascade && (!root || t->first[k] != 0 || t->offset[k] != 0);
        c.mode = paged ? CC_ROWS_NEW : (f & DGX_CASCADE_FILTERED) && !skip ? CC_ROWS_OLD : CC_ROWS_KEEP;
        c.prune = cascade && !skip;
        c.ordered = (f & DGX_CASCADE_ORDERED) != 0;
        c.first = paged ? t->first[k] : 0;
        c.offset = paged ? t->offset[k] : 0;
        c.ck_b = (uint32_t)P->ck.size();
        if (c.prune) P->ck.insert(P->ck.end(), checked[k].begin(), checked[k].end());
        c.ck_e = (uint32_t)P->ck.size();
        P->nv += s.vcap;
        P->no += s.nrows + 1;
        P->nd += s.ndest;
        P->nh += s.nhv;
    }
    for (size_t i = 0; i + 1 < lb.size(); ++i) {
        const CcNode &a = P->node[lb[i]], &z = P->node[lb[i + 1] - 1];
        CcLevel L{};
        L.a = lb[i];
        L.b = lb[i + 1];
        L.va = a.vb;
        L.nv = z.vb + z.vcap - a.vb;
        L.da = a.db;
        L.nd = z.db + z.ndest - a.db;
        L.oa = a.ob;
        L.no = z.ob + z.nrows + 1 - a.ob;
        if (L.nv == 0 && L.nd == 0) continue;  // its rows and dest are empty already
        P->max_nv = std::max<uint64_t>(P->max_nv, L.nv);
        P->max_nd = std::max<uint64_t>(P->max_nd, L.nd);
        P->level.push_back(L);
    }
}

// The whole call on the lane: one metadata copy, 4 + 7 * D launches.  Workspace: 44 bytes per value slot (gathered
// and kept values 16, and a level's flags, their three scans and rows 28), 16 per offset slot, 16 per dest slot plus
// 16 per dest slot of the largest level, 1 per has_val byte, about 140 per node, and the scans' look-back words.
static int cc_run(dgx_lane* l, const CcPlan& T, uint64_t* d_out, uint64_t* d_out_off, uint64_t* d_dest_out,
                  uint64_t* d_dest_off, uint64_t* d_sizes) {
    const uint64_t NN = T.node.size(), D = T.level.size();
    uint64_t nstatus = scan_tiles(2 * NN);
    for (const CcLevel& L : T.level) nstatus += scan_tiles(L.nd) + 2 * scan_tiles(L.nv);
    const uint64_t nscan = 3 * D + 1;
    // copied: the nodes, the checked children and the scans' size words
    CcParams P;
    CcNode* h_node;
    uint32_t* h_ck;
    uint64_t* h_words;
    const u64* d_words;
    u64* status;
    u32* ticket;
    WsCarve ws(l);
    ws.copied(&P.node, &h_node, NN);
    ws.copied(&P.ck, &h_ck, T.ck.size() + 1);
    ws.copied(&d_words, &h_words, 2 * D + 1);
    if (int rc = ws.stage()) return rc;
    memcpy(h_node, T.node.data(), NN * sizeof(CcNode));
    if (!T.ck.empty()) memcpy(h_ck, T.ck.data(), T.ck.size() * sizeof(uint32_t));
    for (uint64_t i = 0; i < D; ++i) {
        h_words[2 * i] = T.level[i].nd;
        h_words[2 * i + 1] = T.level[i].nv;
    }
    h_words[2 * D] = 2 * NN;
    ws.zeroed(&P.bad, 4);
    ws.zeroed(&ticket, nscan);
    ws.zeroed(&status, nstatus);
    ws.plain(&P.V, T.nv);
    ws.plain(&P.OV, T.nv);
    ws.plain(&P.VO, T.no);
    ws.plain(&P.OO, T.no);
    ws.plain(&P.D, T.nd);
    ws.plain(&P.ND, T.nd);
    ws.plain(&P.NDE, NN);
    ws.plain(&P.keep, T.max_nd);
    ws.plain(&P.kx, T.max_nd + 1);
    ws.plain(&P.fv, T.max_nv);
    ws.plain(&P.fx, T.max_nv + 1);
    ws.plain(&P.fy, T.max_nv + 1);
    ws.plain(&P.cnt, 2 * NN);
    ws.plain(&P.cx, 2 * NN + 1);
    ws.plain(&P.rw, T.max_nv);
    ws.plain(&P.H, T.nh);
    if (int rc = ws.commit()) return rc;
    P.nnodes = (u32)NN;
    P.nv = T.nv;
    P.no = T.no;
    P.nd = T.nd;
    P.nh = T.nh;
    P.out_rows = T.rows;
    P.err = l->d_err;
    P.out = (u64*)d_out;
    P.out_off = (u64*)d_out_off;
    P.dest_out = (u64*)d_dest_out;
    P.dest_off = (u64*)d_dest_off;
    P.sizes = (u64*)d_sizes;
    auto scan = [&](const u64* in, u64* out, const u64* n_word, uint64_t n) {
        const uint64_t tiles = scan_tiles(n);
        scan_u64_kernel<<<(unsigned)tiles, EN_NT, 0, l->stream>>>(in, out, n_word, n, status, ticket, nullptr);
        status += tiles;
        ticket += 1;
    };
    cc_gather_kernel<<<gb_grid(std::max<uint64_t>({T.nv, T.no, T.nd, T.nh, NN})), 256, 0, l->stream>>>(P);
    for (uint64_t i = 0; i < D; ++i) {
        CcLevel L = T.level[i];
        L.n_dest = d_words + 2 * i;
        L.n_val = d_words + 2 * i + 1;
        cc_keep_kernel<<<gb_grid(L.nd), 256, 0, l->stream>>>(P, L);
        scan(P.keep, P.kx, L.n_dest, L.nd);
        cc_filter_kernel<<<gb_grid(std::max<uint64_t>({L.nd, L.nv, L.b - L.a})), 256, 0, l->stream>>>(P, L);
        scan(P.fv, P.fx, L.n_val, L.nv);
        cc_page_kernel<<<gb_grid(L.nv), 256, 0, l->stream>>>(P, L);
        scan(P.fv, P.fy, L.n_val, L.nv);
        cc_compact_kernel<<<gb_grid(std::max<uint64_t>(L.nv, L.no)), 256, 0, l->stream>>>(P, L);
    }
    cc_count_kernel<<<gb_grid(NN), 256, 0, l->stream>>>(P);
    scan(P.cnt, P.cx, d_words + 2 * D, 2 * NN);
    cc_place_kernel<<<gb_grid(std::max<uint64_t>({T.nv, T.no, T.nd, NN + 1})), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 4 + 7 * (int)D);
    return DGX_OK;
}

// Sizes and pointers of a planned call, before anything is copied.
static int cc_check_plan(const CcPlan& T, size_t out_cap, size_t dest_cap) {
    if (T.rows >= kCcMax || T.nv >= kCcMax || T.nd >= kCcMax)
        return fail(DGX_ERR_ARG, "cascade sizes are 32-bit: %llu rows, %llu values, %llu dest values in all",
                    (unsigned long long)T.rows, (unsigned long long)T.nv, (unsigned long long)T.nd);
    if (out_cap < T.nv || dest_cap < T.nd)
        return fail(DGX_ERR_CAP, "out_cap %zu / dest_cap %zu below the bounds %llu / %llu", out_cap, dest_cap,
                    (unsigned long long)T.nv, (unsigned long long)T.nd);
    return DGX_OK;
}

extern "C" int dgx_dev_cascade(dgx_lane* l, const dgx_cascade_tree* tree, const dgx_cascade_node* nodes,
                               uint64_t* d_out, uint64_t* d_out_off, size_t out_cap, uint64_t* d_dest_out,
                               uint64_t* d_dest_out_off, size_t dest_cap, uint64_t* d_sizes) {
    if (!l || !d_out_off || !d_dest_out_off || !d_sizes) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = cc_check_tree(tree)) return rc;
    const size_t n = tree->nnodes;
    if (n && !nodes) return fail(DGX_ERR_ARG, "null nodes");
    std::vector<CcSrc> src(n);
    for (size_t k = 0; k < n; ++k) {
        const dgx_cascade_node& c = nodes[k];
        if (!c.v_off || (c.v_cap && !c.v) || (c.ndest && !c.dest) || (c.nhas && !c.has_val))
            return fail(DGX_ERR_ARG, "node %zu: null array", k);
        src[k] = {c.v, c.v_off, 0, c.nrows, c.v_cap, c.dest, c.ndest, c.has_val, c.nhas};
    }
    CcPlan T;
    cc_plan(tree, src.data(), &T);
    if (int rc = cc_check_plan(T, out_cap, dest_cap)) return rc;
    if ((T.nv && !d_out) || (T.nd && !d_dest_out)) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_out_off, (T.rows + 1) * sizeof(uint64_t));
    l->note_output(d_dest_out_off, (n + 1) * sizeof(uint64_t));
    l->note_output(d_sizes, 2 * sizeof(uint64_t));
    if (T.level.empty()) {  // no dest value and no value slot: every row and dest is empty
        CK(cudaMemsetAsync(d_out_off, 0, (T.rows + 1) * sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_dest_out_off, 0, (n + 1) * sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_sizes, 0, 2 * sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (int rc = cc_run(l, T, d_out, d_out_off, d_dest_out, d_dest_out_off, d_sizes)) return rc;
    g_stats.uids_in += T.nv + T.nd;
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_dest_out, dest_cap * sizeof(uint64_t));
    return DGX_OK;
}

extern "C" int dgx_cascade(const dgx_cascade_tree* tree, const uint64_t* v, const uint64_t* v_off,
                           const uint64_t* row_off, const uint64_t* dest, const uint64_t* dest_off,
                           const uint8_t* has_val, const uint64_t* hv_off, uint64_t* out, uint64_t* out_off,
                           size_t out_cap, uint64_t* dest_out, uint64_t* dest_out_off, size_t dest_cap) {
    if (!out_off || !dest_out_off) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = cc_check_tree(tree)) return rc;
    const size_t n = tree->nnodes;
    if (n == 0) {
        out_off[0] = dest_out_off[0] = 0;
        return DGX_OK;
    }
    if (!row_off || !v_off || !dest_off || !hv_off) return fail(DGX_ERR_ARG, "null argument");
    int rc;
    if ((rc = check_offsets("row_off", row_off, n, kCcMax)) || (rc = check_offsets("v_off", v_off, row_off[n], kCcMax)) ||
        (rc = check_offsets("dest_off", dest_off, n, kCcMax)) || (rc = check_offsets("hv_off", hv_off, n, UINT64_MAX)))
        return rc;
    const uint64_t rows = row_off[n], m = v_off[rows], nd = dest_off[n], nh = hv_off[n];
    if ((m && !v) || (nd && !dest) || (nh && !has_val)) return fail(DGX_ERR_ARG, "null argument");
    if ((m && !out) || (nd && !dest_out)) return fail(DGX_ERR_ARG, "null argument");
    if (out_cap < m || dest_cap < nd)
        return fail(DGX_ERR_CAP, "out_cap %zu / dest_cap %zu below the bounds %llu / %llu", out_cap, dest_cap,
                    (unsigned long long)m, (unsigned long long)nd);
    if (m == 0 && nd == 0) {
        memset(out_off, 0, (rows + 1) * sizeof(uint64_t));
        memset(dest_out_off, 0, (n + 1) * sizeof(uint64_t));
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += m + nd;
    uint64_t *d_v, *d_v_off, *d_dest;
    uint8_t* d_hv;
    WsCarve in(l);
    in.plain(&d_hv, nh + 16);
    if ((rc = upload_list(l, v, m, &d_v)) || (rc = upload_list(l, v_off, rows + 1, &d_v_off)) ||
        (rc = upload_list(l, dest, nd, &d_dest)) || (rc = in.commit()))
        return rc;
    if (nh) CK(cudaMemcpyAsync(d_hv, has_val, nh, cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += nh;
    std::vector<CcSrc> src(n);
    for (size_t k = 0; k < n; ++k) {
        const uint64_t r0 = row_off[k], r1 = row_off[k + 1];
        src[k] = {d_v + v_off[r0], d_v_off + r0, v_off[r0], r1 - r0, v_off[r1] - v_off[r0], d_dest + dest_off[k],
                  dest_off[k + 1] - dest_off[k], d_hv + hv_off[k], hv_off[k + 1] - hv_off[k]};
    }
    CcPlan T;
    cc_plan(tree, src.data(), &T);
    if ((rc = cc_check_plan(T, m, nd))) return rc;
    uint64_t *d_sizes, *d_out, *d_dout, *d_ooff, *d_doff;
    WsCarve o(l);
    o.plain(&d_sizes, 2);
    o.plain(&d_out, m);
    o.plain(&d_dout, nd);
    o.plain(&d_ooff, rows + 1);
    o.plain(&d_doff, n + 1);
    if ((rc = o.commit())) return rc;
    if ((rc = cc_run(l, T, d_out, d_ooff, d_dout, d_doff, d_sizes))) return rc;
    CK(cudaMemcpyAsync(l->h_word, d_sizes, 2 * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if ((rc = dgx_lane_sync(l))) return rc;
    const uint64_t K = l->h_word[0], DN = l->h_word[1];
    CK(cudaMemcpyAsync(out_off, d_ooff, (rows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(dest_out_off, d_doff, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (K) CK(cudaMemcpyAsync(out, d_out, K * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (DN) CK(cudaMemcpyAsync(dest_out, d_dout, DN * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += (K + DN + rows + n + 4) * sizeof(uint64_t);
    g_stats.uids_out += K + DN;
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// @filter and first / offset: a subgraph's filter tree over its uid matrix in one call (sg_filter_kernel.cuh)
// ---------------------------------------------------------------------------
constexpr uint64_t kSfMax = uint64_t(1) << 32;  // |D0|, rows, values and list lengths are 32-bit counts

// The checks of the tree and the leaves, and the tree's pre-order program.
static int sf_check_args(const dgx_sg_filter_tree* t, const dgx_sg_filter_leaf* leaves, size_t nleaves, bool dev,
                         std::vector<SfOp>* prog) {
    if (!t) return fail(DGX_ERR_ARG, "null tree");
    const size_t n = t->nnodes;
    if (n == 0 || n > DGX_SGF_MAX_NODES) return fail(DGX_ERR_ARG, "%zu nodes: 1 to %d", n, DGX_SGF_MAX_NODES);
    if (!t->op || !t->parent || !t->leaf) return fail(DGX_ERR_ARG, "null tree array");
    if (nleaves > DGX_SGF_MAX_LEAVES) return fail(DGX_ERR_ARG, "%zu leaves: at most %d", nleaves, DGX_SGF_MAX_LEAVES);
    if (nleaves && !leaves) return fail(DGX_ERR_ARG, "null leaves");
    for (size_t j = 0; j < nleaves; ++j) {
        const dgx_sg_filter_leaf& L = leaves[j];
        if (L.kind == DGX_SGF_LIST) {
            if (L.n >= kSfMax) return fail(DGX_ERR_ARG, "leaf %zu: %zu uids, at most 2^32 - 1", j, L.n);
            if (L.n && !L.uids) return fail(DGX_ERR_ARG, "leaf %zu: null uids", j);
            if (L.d_len && !dev) return fail(DGX_ERR_ARG, "leaf %zu: a length word in the host form", j);
        } else if (L.kind == DGX_SGF_COUNT) {
            if (L.cmp < DGX_SGF_CMP_LE || L.cmp > DGX_SGF_CMP_EQ) return fail(DGX_ERR_ARG, "leaf %zu: cmp %d", j, L.cmp);
            if (!L.counts == !L.off) return fail(DGX_ERR_ARG, "leaf %zu: not exactly one of counts and off", j);
        } else {
            return fail(DGX_ERR_ARG, "leaf %zu: unknown kind %d", j, L.kind);
        }
    }
    std::vector<std::vector<uint32_t>> kids(n);
    std::vector<uint32_t> depth(n, 0);
    for (size_t k = 0; k < n; ++k) {
        const uint8_t op = t->op[k];
        if (op > DGX_SGF_NOT) return fail(DGX_ERR_ARG, "node %zu: unknown op %u", k, (unsigned)op);
        if (op == DGX_SGF_LEAF && t->leaf[k] >= nleaves)
            return fail(DGX_ERR_ARG, "node %zu: leaf %u past %zu leaves", k, t->leaf[k], nleaves);
        if (k == 0) continue;
        const uint32_t p = t->parent[k];
        if (p >= k) return fail(DGX_ERR_ARG, "node %zu: parent %u is not below it", k, p);
        if (t->op[p] == DGX_SGF_LEAF) return fail(DGX_ERR_ARG, "node %zu: its parent %u is a leaf", k, p);
        depth[k] = depth[p] + 1;
        if (depth[k] > DGX_SGF_MAX_DEPTH) return fail(DGX_ERR_ARG, "node %zu is deeper than %d", k, DGX_SGF_MAX_DEPTH);
        kids[p].push_back((uint32_t)k);
    }
    for (size_t k = 0; k < n; ++k) {
        const uint8_t op = t->op[k];
        if (op == DGX_SGF_NOT && kids[k].size() != 1)
            return fail(DGX_ERR_ARG, "node %zu: NOT with %zu children", k, kids[k].size());
        if ((op == DGX_SGF_AND || op == DGX_SGF_OR) && kids[k].empty())
            return fail(DGX_ERR_ARG, "node %zu: AND / OR without children", k);
    }
    // pre-order: a node's entry is written when it is reached, its end once its subtree is
    prog->assign(n, SfOp{0, 0});
    std::vector<std::pair<uint32_t, uint32_t>> stack{{0u, kSfNoParent}};  // (node, parent's entry)
    std::vector<uint32_t> pos(n);
    uint32_t pc = 0;
    while (!stack.empty()) {
        const auto [k, pe] = stack.back();
        stack.pop_back();
        pos[k] = pc;
        const uint8_t op = t->op[k];
        (*prog)[pc++] = op == DGX_SGF_LEAF ? SfOp{t->leaf[k], pe} : SfOp{kSfNode | (uint32_t)op << 28, pe};
        for (size_t c = kids[k].size(); c-- > 0;) stack.push_back({kids[k][c], pos[k]});
    }
    // a subtree's end: one past its last pre-order entry, which is the end of its last child (or itself for a leaf)
    std::vector<uint32_t> end(n);
    for (size_t k = n; k-- > 0;) end[k] = kids[k].empty() ? pos[k] + 1 : end[kids[k].back()];
    for (size_t k = 0; k < n; ++k)
        if (t->op[k] != DGX_SGF_LEAF) (*prog)[pos[k]].w0 |= end[k];
    return DGX_OK;
}

// The whole call on the lane: one table copy, 11 launches.  Workspace: 28 bytes per value slot of v_cap (cascade's
// flags and their two scans, 8 each, and rows, 4), 40 per D0 slot (keep flags and their scan, D1, marks and their
// scan), and the scans' look-back words.  `out` null: counts-only, no row value written.
static int sf_run(dgx_lane* l, const std::vector<SfOp>& prog, const dgx_sg_filter_leaf* leaves, size_t nleaves,
                  const uint64_t* d0, const uint64_t* d0_len, uint64_t d0_cap, const uint64_t* v, const uint64_t* v_off,
                  uint64_t nrows, uint64_t v_cap, int32_t count, int32_t offset, uint64_t* dest_out,
                  uint64_t* dest_len, uint64_t* out, uint64_t* out_off, uint32_t* counts) {
    SfParams S{};
    CcParams P{};
    SfLeaf* h_leaf;
    SfOp* h_prog;
    CcNode* h_node;
    u64* status;
    u32* ticket;
    const uint64_t td = scan_tiles(d0_cap), tv = scan_tiles(v_cap);
    WsCarve ws(l);
    ws.copied(&S.leaf, &h_leaf, std::max<size_t>(nleaves, 1));
    ws.copied(&S.prog, &h_prog, prog.size());
    ws.copied(&S.node, &h_node, 1);
    if (int rc = ws.stage()) return rc;
    uint64_t slots = 0;
    for (size_t j = 0; j < nleaves; ++j) {
        const dgx_sg_filter_leaf& L = leaves[j];
        SfLeaf& s = h_leaf[j];
        s = SfLeaf{};
        s.kind = L.kind == DGX_SGF_LIST ? SF_LIST : SF_COUNT;
        s.sb = slots;
        if (L.kind == DGX_SGF_LIST) {
            s.p = (const u64*)L.uids;
            s.len = (const u64*)L.d_len;
            s.room = L.n;
            slots += L.n + 1;
        } else {
            s.cnt = L.counts;
            s.off = (const u64*)L.off;
            s.cmp = (u32)L.cmp;
            s.thr = L.threshold;
            if (L.off) slots += d0_cap;
        }
    }
    memcpy(h_prog, prog.data(), prog.size() * sizeof(SfOp));
    CcNode& c = *h_node;
    c = CcNode{};
    c.vcap = v_cap;
    c.nrows = nrows;
    c.ndest = d0_cap;  // |D0| once sf_check_kernel has run
    c.mode = CC_ROWS_NEW;
    c.ordered = 1;     // the rows' order is sf_check_kernel's
    c.first = count;
    c.offset = offset;
    ws.zeroed(&S.bad, 4);
    ws.zeroed(&ticket, 4);
    ws.zeroed(&status, 2 * td + 2 * tv);
    ws.zeroed(&S.mark, d0_cap);
    ws.plain(&S.words, 2);
    ws.plain(&P.keep, d0_cap);
    ws.plain(&P.kx, d0_cap + 1);
    ws.plain(&P.ND, d0_cap);
    ws.plain(&P.NDE, 1);
    ws.plain(&P.fv, v_cap);
    ws.plain(&P.fx, v_cap + 1);
    ws.plain(&P.fy, v_cap + 1);
    ws.plain(&P.rw, v_cap);
    u64* mx;
    ws.plain(&mx, d0_cap + 1);
    if (int rc = ws.commit()) return rc;
    S.nleaves = (u32)nleaves;
    S.d0 = (const u64*)d0;
    S.d0_len = (const u64*)d0_len;
    S.d0_cap = d0_cap;
    S.v_off = (const u64*)v_off;
    S.v = (const u64*)v;
    S.nrows = nrows;
    S.v_cap = v_cap;
    S.slots = slots;
    S.counts_only = out == nullptr;
    S.paged = count != 0 || offset != 0;
    S.keep = P.keep;
    S.d1 = P.ND;
    S.n1 = P.NDE;
    S.fv = P.fv;
    S.oo = (const u64*)out_off;
    S.mx = mx;
    S.err = l->d_err;
    S.dest_out = (u64*)dest_out;
    S.dest_len = (u64*)dest_len;
    S.counts = counts;
    // cascade's one NEW node reads the inputs in place (the level kernels never write V, VO or D) and writes the
    // kept values and row offsets straight into the outputs
    P.node = S.node;
    P.nnodes = 1;
    P.nv = v_cap;
    P.no = nrows + 1;
    P.nd = d0_cap;
    P.out_rows = nrows;
    P.V = const_cast<u64*>(S.v);
    P.VO = const_cast<u64*>(S.v_off);
    P.D = const_cast<u64*>(S.d0);
    P.OV = (u64*)out;
    P.OO = (u64*)out_off;
    P.bad = S.bad;
    P.err = l->d_err;
    CcLevel L{};
    L.a = 0;
    L.b = 1;
    L.nv = v_cap;
    L.nd = d0_cap;
    L.no = nrows + 1;
    L.n_dest = S.words;
    L.n_val = S.words + 1;
    CcLevel Lc = L;
    if (S.counts_only) Lc.nv = 0;  // the row offsets only
    auto scan = [&](const u64* in, u64* o, const u64* n_word, uint64_t n) {
        const uint64_t tiles = scan_tiles(n);
        scan_u64_kernel<<<(unsigned)tiles, EN_NT, 0, l->stream>>>(in, o, n_word, n, status, ticket, nullptr);
        status += tiles;
        ticket += 1;
    };
    sf_check_kernel<<<gb_grid(std::max<uint64_t>({d0_cap, slots, nrows + 1, v_cap})), 256, 0, l->stream>>>(S);
    sf_eval_kernel<<<gb_grid(d0_cap), 256, 0, l->stream>>>(S);
    scan(P.keep, P.kx, L.n_dest, d0_cap);
    cc_filter_kernel<<<gb_grid(std::max<uint64_t>({d0_cap, v_cap, 1})), 256, 0, l->stream>>>(P, L);
    scan(P.fv, P.fx, L.n_val, v_cap);
    cc_page_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P, L);
    scan(P.fv, P.fy, L.n_val, v_cap);
    cc_compact_kernel<<<gb_grid(std::max<uint64_t>(Lc.nv, Lc.no)), 256, 0, l->stream>>>(P, Lc);
    sf_mark_kernel<<<gb_grid(std::max<uint64_t>(d0_cap, v_cap)), 256, 0, l->stream>>>(S);
    scan(S.mark, mx, P.NDE, d0_cap);
    sf_out_kernel<<<gb_grid(std::max<uint64_t>(d0_cap, nrows)), 256, 0, l->stream>>>(S);
    CK(cudaGetLastError());
    count_launches(l, 11);
    return DGX_OK;
}

extern "C" int dgx_dev_sg_filter(dgx_lane* l, const dgx_sg_filter_tree* tree, const dgx_sg_filter_leaf* leaves,
                                 size_t nleaves, const uint64_t* d_d0, size_t d0_cap, const uint64_t* d_d0_len,
                                 const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows, size_t v_cap,
                                 int32_t count, int32_t offset, uint64_t* d_dest_out, size_t dest_cap,
                                 uint64_t* d_dest_len, uint64_t* d_out, uint64_t* d_out_off, size_t out_cap,
                                 uint32_t* d_counts) {
    if (!l || !d_dest_len || !d_v_off || !d_out_off || (nrows && !d_counts)) return fail(DGX_ERR_ARG, "null argument");
    std::vector<SfOp> prog;
    if (int rc = sf_check_args(tree, leaves, nleaves, true, &prog)) return rc;
    if (d0_cap >= kSfMax || nrows >= kSfMax || v_cap >= kSfMax)
        return fail(DGX_ERR_ARG, "sizes are 32-bit: d0_cap %zu, nrows %zu, v_cap %zu", d0_cap, nrows, v_cap);
    if ((d0_cap && !d_d0) || (v_cap && !d_v)) return fail(DGX_ERR_ARG, "null argument");
    if (dest_cap < d0_cap || (d_out && out_cap < v_cap))
        return fail(DGX_ERR_CAP, "dest_cap %zu / out_cap %zu below the bounds %zu / %zu", dest_cap, out_cap, d0_cap,
                    v_cap);
    if (d0_cap && !d_dest_out) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_dest_len, sizeof(uint64_t));
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    l->note_output(d_counts, nrows * sizeof(uint32_t));
    if (d0_cap == 0) {  // D0 is empty: so are D1, the rows and the new dest
        CK(cudaMemsetAsync(d_dest_len, 0, sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_out_off, 0, (nrows + 1) * sizeof(uint64_t), l->stream));
        if (nrows) CK(cudaMemsetAsync(d_counts, 0, nrows * sizeof(uint32_t), l->stream));
        return DGX_OK;
    }
    if (int rc = sf_run(l, prog, leaves, nleaves, d_d0, d_d0_len, d0_cap, d_v, d_v_off, nrows, v_cap, count, offset,
                        d_dest_out, d_dest_len, d_out, d_out_off, d_counts))
        return rc;
    g_stats.uids_in += d0_cap + v_cap;
    l->note_output(d_dest_out, dest_cap * sizeof(uint64_t));
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    return DGX_OK;
}

extern "C" int dgx_sg_filter(const dgx_sg_filter_tree* tree, const dgx_sg_filter_leaf* leaves, size_t nleaves,
                             const uint64_t* d0, size_t n0, const uint64_t* v, const uint64_t* v_off, size_t nrows,
                             int32_t count, int32_t offset, uint64_t* dest_out, size_t dest_cap, size_t* dest_len,
                             uint64_t* out, uint64_t* out_off, size_t out_cap, uint32_t* counts) {
    if (!dest_len || !v_off || !out_off || (nrows && !counts)) return fail(DGX_ERR_ARG, "null argument");
    std::vector<SfOp> prog;
    int rc;
    if ((rc = sf_check_args(tree, leaves, nleaves, false, &prog))) return rc;
    if (n0 >= kSfMax || nrows >= kSfMax)
        return fail(DGX_ERR_ARG, "sizes are 32-bit: n0 %zu, nrows %zu", n0, nrows);
    if ((rc = check_offsets("v_off", v_off, nrows, kSfMax))) return rc;
    const uint64_t m = v_off[nrows];
    if ((n0 && !d0) || (m && !v)) return fail(DGX_ERR_ARG, "null argument");
    if (dest_cap < n0 || (out && out_cap < m))
        return fail(DGX_ERR_CAP, "dest_cap %zu / out_cap %zu below the bounds %zu / %llu", dest_cap, out_cap, n0,
                    (unsigned long long)m);
    if (n0 && !dest_out) return fail(DGX_ERR_ARG, "null argument");
    if (n0 == 0) {  // D0 is empty: so are D1, the rows and the new dest
        *dest_len = 0;
        memset(out_off, 0, (nrows + 1) * sizeof(uint64_t));
        if (nrows) memset(counts, 0, nrows * sizeof(uint32_t));
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += n0 + m;
    std::vector<dgx_sg_filter_leaf> D(leaves, leaves + nleaves);  // one copy of each array
    uint64_t *d_d0, *d_v, *d_v_off;
    if ((rc = upload_list(l, d0, n0, &d_d0)) || (rc = upload_list(l, v, m, &d_v)) ||
        (rc = upload_list(l, v_off, nrows + 1, &d_v_off)))
        return rc;
    for (dgx_sg_filter_leaf& L : D) {
        uint64_t* p;
        if (L.kind == DGX_SGF_LIST) {
            if ((rc = upload_list(l, L.uids, L.n, &p))) return rc;
            L.uids = p;
            g_stats.uids_in += L.n;
        } else if (L.off) {
            if ((rc = upload_list(l, L.off, n0 + 1, &p))) return rc;
            L.off = p;
        } else {
            void* q;
            if ((rc = l->ws.alloc(n0 * sizeof(uint32_t) + 16, &q))) return rc;
            CK(cudaMemcpyAsync(q, L.counts, n0 * sizeof(uint32_t), cudaMemcpyHostToDevice, l->stream));
            g_stats.h2d += n0 * sizeof(uint32_t);
            L.counts = (const uint32_t*)q;
        }
    }
    uint64_t *o_len, *o_dest, *o_out = nullptr, *o_off;
    uint32_t* o_counts;
    WsCarve o(l);
    o.plain(&o_len, 2);
    o.plain(&o_dest, n0);
    if (out) o.plain(&o_out, m);
    o.plain(&o_off, nrows + 1);
    o.plain(&o_counts, nrows + 1);
    if ((rc = o.commit())) return rc;
    if ((rc = sf_run(l, prog, D.data(), nleaves, d_d0, nullptr, n0, d_v, d_v_off, nrows, m, count, offset, o_dest,
                     o_len, o_out, o_off, o_counts)))
        return rc;
    CK(cudaMemcpyAsync(l->h_word, o_len, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(l->h_word + 1, o_off + nrows, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if ((rc = dgx_lane_sync(l))) return rc;
    const uint64_t DN = l->h_word[0], K = l->h_word[1];
    *dest_len = DN;
    CK(cudaMemcpyAsync(out_off, o_off, (nrows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (nrows) CK(cudaMemcpyAsync(counts, o_counts, nrows * sizeof(uint32_t), cudaMemcpyDeviceToHost, l->stream));
    if (DN) CK(cudaMemcpyAsync(dest_out, o_dest, DN * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (out && K) CK(cudaMemcpyAsync(out, o_out, K * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += (DN + (out ? K : 0) + nrows + 3) * sizeof(uint64_t) + nrows * sizeof(uint32_t);
    g_stats.uids_out += DN + (out ? K : 0);
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// orderasc / orderdesc by a value variable: a uid matrix sorted in Go's exact order and paged (var_order_kernel.cuh)
// ---------------------------------------------------------------------------
constexpr uint64_t kVoMax = uint64_t(1) << 32;  // dest, map, rows and values are 32-bit counts

// The row sort's radix passes, from nrows alone: P_r = ceil(bits(nrows - 1) / 8).
static uint32_t vo_row_passes(uint64_t nrows) {
    return (gb_bits(nrows ? nrows - 1 : 0) + GB_DIGIT_BITS - 1) / GB_DIGIT_BITS;
}

// The checks of the map both forms make before anything is copied.
static int vo_check_var(const dgx_math_leaf* var, bool dev) {
    if (!var) return fail(DGX_ERR_ARG, "null map");
    if (var->nil) return fail(DGX_ERR_ARG, "the variable has no map: used before definition");
    if (!var->tag && var->type != DGX_VAL_INT64 && var->type != DGX_VAL_FLOAT64)
        return fail(DGX_ERR_ARG, "a map without tags has type DGX_VAL_INT64 or DGX_VAL_FLOAT64, not %d", var->type);
    if (!dev && var->d_len) return fail(DGX_ERR_ARG, "d_len belongs to the device form");
    if (var->n >= kVoMax) return fail(DGX_ERR_ARG, "a map of 2^32 entries or more");
    if (var->n && (!var->key || !var->word)) return fail(DGX_ERR_ARG, "null map array");
    return DGX_OK;
}

// The whole call on the lane: 37 + 3 P_r launches.  Workspace: words, tickets and the look-back words, zeroed; per
// value slot of v_cap about 120 bytes (U and W flags and their scans 32, map index 4, U 8, W's uids, words, tags and
// rows 21, order keys 8, radix keys and payloads 24, pair slots 4, the radix hist); per row 44 (offsets of U and W,
// flags, list, page start, page length and its scan); 16 per dest slot (marks and their scan).
static int vo_run(dgx_lane* l, const dgx_math_leaf& M, int desc, const uint64_t* dest, const uint64_t* dlen,
                  uint64_t dcap, const uint64_t* v, const uint64_t* v_off, uint64_t nrows, uint64_t v_cap,
                  int32_t count, int32_t offset, uint64_t* out, uint64_t* out_off, uint64_t* dest_out,
                  uint64_t* dest_len) {
    const uint64_t vc = std::max<uint64_t>(v_cap, 1), tv = scan_tiles(vc), tr = scan_tiles(nrows), td = scan_tiles(dcap);
    const uint64_t tiles = (vc + GB_TILE - 1) / GB_TILE, hn = (uint64_t)GB_RADIX * tiles, th = scan_tiles(hn);
    const uint32_t pr = vo_row_passes(nrows);
    VoParams P{};
    u64 *status, *ek[2], *hist, *hoff;
    u32 *tickets, *ep[2];
    WsCarve ws(l);
    ws.zeroed(&P.bad, 4);
    ws.zeroed(&P.words, VO_WORDS);
    ws.zeroed(&tickets, 32);
    ws.zeroed(&status, 2 * tv + (VO_KEY_PASSES + pr) * th + tr + td);
    ws.zeroed(&P.rflag, nrows);
    ws.zeroed(&P.mark, dcap);
    ws.plain(&P.uf, vc);
    ws.plain(&P.ux, vc + 1);
    ws.plain(&P.wf, vc);
    ws.plain(&P.wx, vc + 1);
    ws.plain(&P.U, vc);
    ws.plain(&P.wuid, vc);
    ws.plain(&P.wword, vc);
    ws.plain(&P.okey, vc);
    ws.plain(&ek[0], vc);
    ws.plain(&ek[1], vc);
    ws.plain(&hist, hn);
    ws.plain(&hoff, hn + 1);
    ws.plain(&P.uoff, nrows + 1);
    ws.plain(&P.woff, nrows + 1);
    ws.plain(&P.plen, nrows);
    ws.plain(&P.po, nrows + 1);
    ws.plain(&P.mx, dcap + 1);
    ws.plain(&P.mj, vc);
    ws.plain(&P.wrow, vc);
    ws.plain(&ep[0], vc);
    ws.plain(&ep[1], vc);
    ws.plain(&P.pairs, vc);
    ws.plain(&P.longrows, nrows);
    ws.plain(&P.pstart, nrows);
    ws.plain(&P.wtag, vc);
    if (int rc = ws.commit()) return rc;
    P.key = (const u64*)M.key;
    P.word = (const u64*)M.word;
    P.tag = M.tag;
    P.mlen = (const u64*)M.d_len;
    P.mcap = M.n;
    P.mtype = M.tag ? 0 : (u32)M.type;
    P.desc = desc != 0;
    P.dest = (const u64*)dest;
    P.dlen = (const u64*)dlen;
    P.dcap = dcap;
    P.v = (const u64*)v;
    P.v_off = (const u64*)v_off;
    P.nrows = nrows;
    P.v_cap = v_cap;
    P.count = count;
    P.offset = offset;
    P.tiles = tiles;
    P.err = l->d_err;
    P.ticket = tickets + 31;
    P.ek = ek[0];
    P.ep = ep[0];
    P.out = (u64*)out;
    P.out_off = (u64*)out_off;
    P.dest_out = (u64*)dest_out;
    P.dest_len = (u64*)dest_len;
    u32* ticket = tickets;
    auto scan = [&](const u64* in, u64* o, const u64* n_word, uint64_t n, u64* total) {
        const uint64_t t = scan_tiles(n);
        scan_u64_kernel<<<(unsigned)t, EN_NT, 0, l->stream>>>(in, o, n_word, n, status, ticket, total);
        status += t;
        ticket += 1;
    };
    vo_check_kernel<<<gb_grid(std::max<uint64_t>({dcap, M.n, nrows + 1, v_cap})), 256, 0, l->stream>>>(P);
    vo_gather_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P);
    scan(P.uf, P.ux, P.words + VO_W_M, vc, nullptr);
    scan(P.wf, P.wx, P.words + VO_W_M, vc, P.words + VO_W_W);
    vo_compact_kernel<<<gb_grid(std::max<uint64_t>(v_cap, nrows + 1)), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 5);
    // W by order key (64 bits: the result is back in buffer 0), then stably by row
    if (int rc = gb_sort(l, tiles, P.bad, P.words + VO_W_H, ek, ep, P.words + VO_W_W, VO_KEY_PASSES, hist, hoff, status,
                         ticket))
        return rc;
    vo_rowkey_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P, ep[0], ek[1], ep[1]);
    u64* const rk[2] = {ek[1], ek[0]};
    u32* const rp[2] = {ep[1], ep[0]};
    if (int rc = gb_sort(l, tiles, P.bad, P.words + VO_W_H, rk, rp, P.words + VO_W_W, pr, hist, hoff, status, ticket))
        return rc;
    P.S = rp[pr & 1];
    vo_tier_kernel<<<gb_grid(std::max<uint64_t>(v_cap, nrows)), 256, 0, l->stream>>>(P);
    vo_rows_kernel<<<gb_grid(nrows), 256, 0, l->stream>>>(P);
    vo_cta_kernel<<<(unsigned)(2 * g_num_sms), VO_NT, 0, l->stream>>>(P);
    scan(P.plen, P.po, P.words + VO_W_R, nrows, nullptr);
    vo_write_kernel<<<gb_grid(std::max<uint64_t>(v_cap, nrows + 1)), 256, 0, l->stream>>>(P);
    scan(P.mark, P.mx, P.words + VO_W_ND, dcap, nullptr);
    vo_dest_kernel<<<gb_grid(dcap), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 8);
    return DGX_OK;
}

extern "C" int dgx_dev_var_order(dgx_lane* l, const dgx_math_leaf* var, int desc, const uint64_t* d_dest, size_t ndest,
                                 const uint64_t* d_ndest, const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows,
                                 size_t v_cap, int32_t count, int32_t offset, uint64_t* d_out, uint64_t* d_out_off,
                                 size_t out_cap, uint64_t* d_dest_out, size_t dest_cap, uint64_t* d_dest_len) {
    if (!l || !d_dest_len || !d_v_off || !d_out_off) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = vo_check_var(var, true)) return rc;
    if (ndest >= kVoMax || nrows >= kVoMax || v_cap >= kVoMax)
        return fail(DGX_ERR_ARG, "sizes are 32-bit: ndest %zu, nrows %zu, v_cap %zu", ndest, nrows, v_cap);
    if ((ndest && !d_dest) || (v_cap && !d_v)) return fail(DGX_ERR_ARG, "null argument");
    if (out_cap < v_cap || dest_cap < ndest)
        return fail(DGX_ERR_CAP, "out_cap %zu / dest_cap %zu below the bounds %zu / %zu", out_cap, dest_cap, v_cap,
                    ndest);
    if ((v_cap && !d_out) || (ndest && !d_dest_out)) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_dest_len, sizeof(uint64_t));
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    if (ndest == 0 || nrows == 0) {  // no dest value or no row: every row is empty, so is the new dest
        CK(cudaMemsetAsync(d_dest_len, 0, sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_out_off, 0, (nrows + 1) * sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (int rc = vo_run(l, *var, desc, d_dest, d_ndest, ndest, d_v, d_v_off, nrows, v_cap, count, offset, d_out,
                        d_out_off, d_dest_out, d_dest_len))
        return rc;
    g_stats.uids_in += ndest + v_cap + var->n;
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_dest_out, dest_cap * sizeof(uint64_t));
    return DGX_OK;
}

extern "C" int dgx_var_order(const dgx_math_leaf* var, int desc, const uint64_t* dest, size_t ndest,
                             const uint64_t* v, const uint64_t* v_off, size_t nrows, int32_t count, int32_t offset,
                             uint64_t* out, uint64_t* out_off, size_t out_cap, uint64_t* dest_out, size_t dest_cap,
                             size_t* dest_len) {
    if (!dest_len || !v_off || !out_off) return fail(DGX_ERR_ARG, "null argument");
    int rc;
    if ((rc = vo_check_var(var, false))) return rc;
    if (ndest >= kVoMax || nrows >= kVoMax) return fail(DGX_ERR_ARG, "sizes are 32-bit: ndest %zu, nrows %zu", ndest, nrows);
    if ((rc = check_offsets("v_off", v_off, nrows, kVoMax))) return rc;
    const uint64_t m = v_off[nrows];
    if ((ndest && !dest) || (m && !v)) return fail(DGX_ERR_ARG, "null argument");
    if (out_cap < m || dest_cap < ndest)
        return fail(DGX_ERR_CAP, "out_cap %zu / dest_cap %zu below the bounds %llu / %zu", out_cap, dest_cap,
                    (unsigned long long)m, ndest);
    if ((m && !out) || (ndest && !dest_out)) return fail(DGX_ERR_ARG, "null argument");
    if (ndest == 0 || nrows == 0) {  // no dest value or no row: every row is empty, so is the new dest
        *dest_len = 0;
        memset(out_off, 0, (nrows + 1) * sizeof(uint64_t));
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += ndest + m + var->n;
    dgx_math_leaf D = *var;  // one copy of each array
    uint64_t *d_dest, *d_v, *d_v_off, *k, *w;
    if ((rc = upload_list(l, dest, ndest, &d_dest)) || (rc = upload_list(l, v, m, &d_v)) ||
        (rc = upload_list(l, v_off, nrows + 1, &d_v_off)) || (rc = upload_list(l, var->key, var->n, &k)) ||
        (rc = upload_list(l, var->word, var->n, &w)))
        return rc;
    D.key = k;
    D.word = w;
    if (var->tag) {
        void* t;
        if ((rc = l->ws.alloc(var->n + 1, &t))) return rc;
        if (var->n) CK(cudaMemcpyAsync(t, var->tag, var->n, cudaMemcpyHostToDevice, l->stream));
        g_stats.h2d += var->n;
        D.tag = (const uint8_t*)t;
    }
    uint64_t *o_len, *o_dest, *o_out, *o_off;
    WsCarve o(l);
    o.plain(&o_len, 1);
    o.plain(&o_dest, ndest);
    o.plain(&o_out, m);
    o.plain(&o_off, nrows + 1);
    if ((rc = o.commit())) return rc;
    if ((rc = vo_run(l, D, desc, d_dest, nullptr, ndest, d_v, d_v_off, nrows, m, count, offset, o_out, o_off, o_dest,
                     o_len)))
        return rc;
    CK(cudaMemcpyAsync(l->h_word, o_len, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(l->h_word + 1, o_off + nrows, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if ((rc = dgx_lane_sync(l))) {
        *dest_len = 0;
        return rc;
    }
    const uint64_t DN = l->h_word[0], K = l->h_word[1];
    *dest_len = DN;
    CK(cudaMemcpyAsync(out_off, o_off, (nrows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (DN) CK(cudaMemcpyAsync(dest_out, o_dest, DN * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (K) CK(cudaMemcpyAsync(out, o_out, K * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += (DN + K + nrows + 3) * sizeof(uint64_t);
    g_stats.uids_out += DN + K;
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// shortest() without weights: one expansion level of every exec sg, the search kept in HBM (path_kernel.cuh)
// ---------------------------------------------------------------------------
constexpr uint64_t kPsMax = uint64_t(1) << 32;  // sgs, rows, values, dest values and set sizes are 32-bit counts

// Seen buffer b holds uid[] at sbuf[b], parent[] at + 8 scap, attr[] at + 16 scap and level[] at + 20 scap bytes;
// expanded buffer b is ebuf[b].  The current buffers, the sizes, the level count and To's level are device words
// (d_state); st mirrors them as of the last wait.  sbound / ebound are the sizes then plus, for every level queued
// since, its bound on new nodes (min(v_cap, dest_cap): a new node is a distinct dest value) and its src_cap, which size
// the capacities without a round trip.
struct dgx_path_search {
    std::mutex mu;
    int device = 0;
    char* sbuf[2] = {nullptr, nullptr};
    uint64_t* ebuf[2] = {nullptr, nullptr};
    uint64_t scap = 0, ecap = 0;
    uint64_t* d_state = nullptr;
    uint64_t st[PS_STATE] = {};
    uint64_t sbound = 0, ebound = 0;
    dgx_lane* lane = nullptr;    // the lane of the device-form levels queued since the last wait
    std::vector<void*> retired;  // buffers replaced by growth, still read by queued levels until the next wait
};

static void ps_free_retired(dgx_path_search* s) {
    for (void* p : s->retired) cudaFree(p);
    s->retired.clear();
}

// Waits for the search's queued levels and reads its words back.  Caller holds s->mu.
static int ps_wait(dgx_path_search* s) {
    CK(cudaSetDevice(s->device));
    if (!s->lane) return DGX_OK;
    CK(cudaMemcpyAsync(s->lane->h_word, s->d_state, sizeof(s->st), cudaMemcpyDeviceToHost, s->lane->stream));
    CK(cudaStreamSynchronize(s->lane->stream));
    memcpy(s->st, s->lane->h_word, sizeof(s->st));
    s->sbound = s->st[PS_S_N];
    s->ebound = s->st[PS_E_N];
    s->lane = nullptr;
    ps_free_retired(s);
    return DGX_OK;
}

// Capacity for `need` records of `rec` bytes (columns of the given widths, each cap records long) in both buffers of a
// ping-pong pair: they grow geometrically, their first `bound` records copied on the stream (the current buffer is only
// known on the device while levels are queued).  The new buffers replace the old ones only once every copy is queued,
// so an allocation or a copy that fails leaves the search as it was.
static int ps_reserve(dgx_path_search* s, cudaStream_t stream, void** buf, uint64_t* cap, uint64_t need,
                      std::initializer_list<size_t> cols, uint64_t bound, uint64_t cur, const char* what) {
    if (need <= *cap) return DGX_OK;
    const uint64_t ncap = std::max(need, 2 * *cap);
    size_t rec = 0;
    for (size_t c : cols) rec += c;
    void* nb[2] = {nullptr, nullptr};
    auto drop = [&](int code, const char* op) {
        cudaGetLastError();
        for (void* p : nb) if (p) cudaFree(p);
        return fail(code, "shortest-path %s growth to %llu records: %s failed", what, (unsigned long long)ncap, op);
    };
    for (int b = 0; b < 2; ++b)
        if (cudaMalloc(&nb[b], ncap * rec) != cudaSuccess) return drop(DGX_ERR_OOM, "cudaMalloc");
    for (int b = 0; b < 2; ++b)
        if (bound && (s->lane || (uint64_t)b == cur)) {  // an idle search's other buffer holds nothing live
            size_t off = 0;
            for (size_t c : cols) {
                if (cudaMemcpyAsync((char*)nb[b] + off * ncap, (char*)buf[b] + off * *cap, bound * c,
                                    cudaMemcpyDeviceToDevice, stream) != cudaSuccess) {
                    if (stream) cudaStreamSynchronize(stream);  // copies already queued read and write nb
                    return drop(DGX_ERR_CUDA, "cudaMemcpyAsync");
                }
                off += c;
            }
        }
    for (int b = 0; b < 2; ++b) {
        if (buf[b]) s->retired.push_back(buf[b]);
        buf[b] = nb[b];
    }
    *cap = ncap;
    return DGX_OK;
}

static int ps_reserve_all(dgx_path_search* s, cudaStream_t stream, uint64_t seen, uint64_t expanded) {
    if (int rc = ps_reserve(s, stream, (void**)s->sbuf, &s->scap, seen, {8, 8, 4, 4}, s->sbound, s->st[PS_S_CUR], "seen"))
        return rc;
    return ps_reserve(s, stream, (void**)s->ebuf, &s->ecap, expanded, {8}, s->ebound, s->st[PS_E_CUR], "expanded");
}

extern "C" int dgx_path_create(uint64_t from, uint64_t to, dgx_path_search** ps) {
    if (!ps) return fail(DGX_ERR_ARG, "null argument");
    if (from == 0 || to == 0 || from == to)
        return fail(DGX_ERR_ARG, "from %llu / to %llu: both nonzero and distinct", (unsigned long long)from,
                    (unsigned long long)to);
    if (int rc = dgx_init(-1)) return rc;
    CK(cudaSetDevice(g_device));
    dgx_path_search* s = new dgx_path_search();
    s->device = g_device;
    s->st[PS_S_N] = 1;
    s->st[PS_TO] = to;
    int rc = DGX_OK;
    if (cudaMalloc(&s->d_state, sizeof(s->st)) != cudaSuccess) rc = fail(DGX_ERR_OOM, "path search allocation failed");
    if (!rc) rc = ps_reserve_all(s, nullptr, 1024, 1024);
    const uint64_t zero[2] = {0, 0};  // From's parent, and its attr and level as two u32
    if (!rc && (cudaMemcpy(s->sbuf[0], &from, 8, cudaMemcpyHostToDevice) != cudaSuccess ||
                cudaMemcpy(s->sbuf[0] + 8 * s->scap, zero, 8, cudaMemcpyHostToDevice) != cudaSuccess ||
                cudaMemcpy(s->sbuf[0] + 16 * s->scap, zero, 4, cudaMemcpyHostToDevice) != cudaSuccess ||
                cudaMemcpy(s->sbuf[0] + 20 * s->scap, zero, 4, cudaMemcpyHostToDevice) != cudaSuccess ||
                cudaMemcpy(s->d_state, s->st, sizeof(s->st), cudaMemcpyHostToDevice) != cudaSuccess))
        rc = fail(DGX_ERR_CUDA, "path search upload failed");
    ps_free_retired(s);
    s->sbound = 1;
    if (rc) {
        dgx_path_destroy(s);
        return rc;
    }
    *ps = s;
    return DGX_OK;
}

extern "C" void dgx_path_destroy(dgx_path_search* s) {
    if (!s) return;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        ps_wait(s);
        ps_free_retired(s);
        for (char* b : s->sbuf) if (b) cudaFree(b);
        for (uint64_t* b : s->ebuf) if (b) cudaFree(b);
        if (s->d_state) cudaFree(s->d_state);
    }
    delete s;
}

// One level on the lane, for a search with room for sbound + min(v_cap, d_cap) seen nodes and ebound + r_cap expanded
// sources: 5 launches, the two matrix merges', 6 launches.  Workspace: 52 bytes per value of v_cap (row and sg 8, new
// flag and position 16, new value 8, N 8, parent 8, sg index 4), 40 per row, 16 per dest value, 8 per sg, the merges'
// about 22 per value of their caps, and the scans' look-back words.  d_next, d_next_off and d_stats are written by the kernels.
static int ps_level(dgx_lane* l, dgx_path_search* s, size_t nsg, const uint32_t* d_attr, const uint64_t* d_src_off,
                    const uint64_t* d_src, uint64_t r_cap, const uint64_t* d_v_off, const uint64_t* d_v, uint64_t v_cap,
                    const uint64_t* d_dest_off, const uint64_t* d_dest, uint64_t d_cap, uint64_t* d_next,
                    uint64_t* d_next_off, uint64_t* d_stats) {
    const uint64_t vc = std::max<uint64_t>(v_cap, 1), rc1 = std::max<uint64_t>(r_cap, 1), dc = std::max<uint64_t>(d_cap, 1);
    auto tiles = [](uint64_t n) { return (n + EN_TILE - 1) / EN_TILE; };
    const uint64_t tv = tiles(vc), tr = tiles(rc1), td = tiles(dc);
    PsParams P;
    u64* status;
    u32* tickets;
    WsCarve ws(l);
    ws.zeroed(&P.bad, 4);
    ws.zeroed(&P.words, PS_WORDS);
    ws.zeroed(&tickets, 10);
    ws.zeroed(&status, tv + tr + td);
    ws.zeroed(&P.rflag, r_cap + 1);
    ws.zeroed(&P.nsgi, vc);
    ws.ones(&P.npar, vc);
    ws.plain(&P.vflag, vc);
    ws.plain(&P.vpos, vc + 1);
    ws.plain(&P.rpos, r_cap + 2);
    ws.plain(&P.nv, vc);
    ws.plain(&P.nv_off, r_cap + 2);
    ws.plain(&P.es, r_cap + 1);
    ws.plain(&P.es_off, nsg + 1);
    ws.plain(&P.nn, vc);
    ws.plain(&P.ne, r_cap + 1);
    ws.plain(&P.dflag, dc);
    ws.plain(&P.dpos, dc + 1);
    ws.plain(&P.vrow, vc);
    ws.plain(&P.vsg, vc);
    if (int rc = ws.commit()) return rc;
    P.nsg = nsg;
    P.attr = (const u32*)d_attr;
    P.src_off = (const u64*)d_src_off;
    P.src = (const u64*)d_src;
    P.r_cap = r_cap;
    P.v_off = (const u64*)d_v_off;
    P.v = (const u64*)d_v;
    P.v_cap = v_cap;
    P.dest_off = (const u64*)d_dest_off;
    P.dest = (const u64*)d_dest;
    P.d_cap = d_cap;
    for (int b = 0; b < 2; ++b) {
        P.su[b] = (u64*)s->sbuf[b];
        P.sp[b] = (u64*)(s->sbuf[b] + 8 * s->scap);
        P.sa[b] = (u32*)(s->sbuf[b] + 16 * s->scap);
        P.sl[b] = (u32*)(s->sbuf[b] + 20 * s->scap);
        P.ex[b] = (u64*)s->ebuf[b];
    }
    P.state = (u64*)s->d_state;
    P.next = (u64*)d_next;
    P.next_off = (u64*)d_next_off;
    P.stats = (u64*)d_stats;
    P.err = l->d_err;
    ps_check_kernel<<<gb_grid(std::max<uint64_t>({nsg + 1, r_cap + 1, v_cap, d_cap})), 256, 0, l->stream>>>(P);
    ps_flags_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)tv, EN_NT, 0, l->stream>>>(P.vflag, P.vpos, P.words + PS_W_M, v_cap, status, tickets,
                                                           P.words + PS_W_NV);
    scan_u64_kernel<<<(unsigned)tr, EN_NT, 0, l->stream>>>(P.rflag, P.rpos, P.words + PS_W_R, r_cap, status + tv,
                                                           tickets + 1, P.words + PS_W_NR);
    ps_gather_kernel<<<gb_grid(std::max<uint64_t>({v_cap, r_cap + 2, nsg + 1})), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 5);
    auto U = [](u64* q) { return (uint64_t*)q; };
    int rc;
    if ((rc = merge_matrix_impl(l, U(P.nv), U(P.nv_off), rc1, vc, U(P.nn), vc, U(P.words + PS_W_NN))) ||
        (rc = merge_matrix_impl(l, U(P.es), U(P.es_off), nsg, rc1, U(P.ne), rc1, U(P.words + PS_W_NE))))
        return rc;
    ps_parent_kernel<<<gb_grid(std::max<uint64_t>(v_cap, d_cap)), 256, 0, l->stream>>>(P);
    ps_attr_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)td, EN_NT, 0, l->stream>>>(P.dflag, P.dpos, P.words + PS_W_D, d_cap,
                                                           status + tv + tr, tickets + 2, P.words + PS_W_NX);
    ps_insert_kernel<<<stride_grid(), 256, 0, l->stream>>>(P);
    ps_write_kernel<<<gb_grid(std::max<uint64_t>(d_cap, nsg + 1)), 256, 0, l->stream>>>(P);
    ps_commit_kernel<<<1, 1, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 6);
    return DGX_OK;
}

// The checks both forms make before anything is copied.  Caller holds s->mu.
static int ps_check_level(dgx_path_search* s, const dgx_lane* l, size_t nsg, uint64_t rows, uint64_t values,
                          uint64_t dests, size_t next_cap) {
    const uint64_t fresh = std::min(values, dests);  // new nodes are distinct dest values
    if (s->lane && s->lane != l)
        return fail(DGX_ERR_ARG, "the path search has levels queued on another lane: wait for them with dgx_path_result");
    if (nsg == 0 || nsg >= kPsMax || rows >= kPsMax || values >= kPsMax || dests >= kPsMax)
        return fail(DGX_ERR_ARG, "shortest-path sizes are 32-bit: 1 to 2^32 - 1 sgs, rows, values and dests below 2^32");
    if (s->sbound + fresh >= kPsMax || s->ebound + rows >= kPsMax)
        return fail(DGX_ERR_ARG, "the path search could reach %llu nodes: at most 2^32 - 1",
                    (unsigned long long)(s->sbound + fresh));
    if (next_cap < dests)
        return fail(DGX_ERR_CAP, "next_cap %zu below the %llu dest values", next_cap, (unsigned long long)dests);
    return DGX_OK;
}

extern "C" int dgx_dev_path_expand(dgx_lane* l, dgx_path_search* s, const dgx_path_level* L, size_t src_cap,
                                   size_t v_cap, size_t dest_cap, uint64_t* d_next, uint64_t* d_next_off,
                                   size_t next_cap, uint64_t* d_stats) {
    if (!l || !s || !L || !d_stats || !d_next_off || !L->attr || !L->src_off || !L->v_off || !L->dest_off ||
        (src_cap && !L->src) || (v_cap && !L->v) || (dest_cap && (!L->dest || !d_next)))
        return fail(DGX_ERR_ARG, "null argument");
    std::lock_guard<std::mutex> lk(s->mu);
    if (int rc = ps_check_level(s, l, L->nsg, src_cap, v_cap, dest_cap, next_cap)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    const uint64_t fresh = std::min<uint64_t>(v_cap, dest_cap);
    if (int rc = ps_reserve_all(s, l->stream, s->sbound + fresh, s->ebound + src_cap)) return rc;
    s->lane = l;  // queued copies or levels now read the search
    s->sbound += fresh;
    s->ebound += src_cap;
    if (int rc = ps_level(l, s, L->nsg, L->attr, L->src_off, L->src, src_cap, L->v_off, L->v, v_cap, L->dest_off,
                          L->dest, dest_cap, d_next, d_next_off, d_stats))
        return rc;
    g_stats.uids_in += v_cap;
    l->note_output(d_next, next_cap * sizeof(uint64_t));
    l->note_output(d_next_off, (L->nsg + 1) * sizeof(uint64_t));
    l->note_output(d_stats, 3 * sizeof(uint64_t));
    return DGX_OK;
}

extern "C" int dgx_path_expand(dgx_path_search* s, const dgx_path_level* L, uint64_t* next, uint64_t* next_off,
                               size_t next_cap, dgx_path_stats* stats) {
    if (!L || !next_off || !stats || !L->attr || !L->src_off || !L->dest_off) return fail(DGX_ERR_ARG, "null argument");
    const size_t S = L->nsg;
    if (S == 0 || S >= kPsMax) return fail(DGX_ERR_ARG, "nsg of %zu: 1 to 2^32 - 1", S);
    if (int rc = check_offsets("src_off", L->src_off, S, kPsMax)) return rc;
    if (int rc = check_offsets("dest_off", L->dest_off, S, kPsMax)) return rc;
    const uint64_t R = L->src_off[S], D = L->dest_off[S];
    if (R && (!L->src || !L->v_off)) return fail(DGX_ERR_ARG, "null argument");
    if (R) if (int rc = check_offsets("v_off", L->v_off, R, kPsMax)) return rc;
    const uint64_t M = R ? L->v_off[R] : 0;
    if ((M && !L->v) || (D && (!L->dest || !next))) return fail(DGX_ERR_ARG, "null argument");
    if (R >= kPsMax || M >= kPsMax || D >= kPsMax) return fail(DGX_ERR_ARG, "shortest-path sizes are 32-bit");
    if (next_cap < D) return fail(DGX_ERR_CAP, "next_cap %zu below the %llu dest values", next_cap, (unsigned long long)D);
    if (!s) return fail(DGX_ERR_ARG, "null path search");  // the level's own errors are reported first
    std::lock_guard<std::mutex> lk(s->mu);
    if (int rc = ps_check_level(s, nullptr, S, R, M, D, next_cap)) return rc;
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += R + M + D;
    static const uint64_t zero = 0;
    uint64_t *d_src_off, *d_src, *d_v_off, *d_v, *d_dest_off, *d_dest, *d_stats, *d_next;
    uint32_t* d_attr;
    WsCarve o(l);
    o.plain(&d_attr, S);
    o.plain(&d_stats, 3 + S + 1);  // stats, then next_off: read back in one copy
    o.plain(&d_next, D + 1);
    int rc;
    if ((rc = upload_list(l, L->src_off, S + 1, &d_src_off)) || (rc = upload_list(l, L->src, R, &d_src)) ||
        (rc = upload_list(l, R ? L->v_off : &zero, R + 1, &d_v_off)) || (rc = upload_list(l, L->v, M, &d_v)) ||
        (rc = upload_list(l, L->dest_off, S + 1, &d_dest_off)) || (rc = upload_list(l, L->dest, D, &d_dest)) ||
        (rc = o.commit()))
        return rc;
    CK(cudaMemcpyAsync(d_attr, L->attr, S * sizeof(uint32_t), cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += S * sizeof(uint32_t);
    uint64_t* d_next_off = d_stats + 3;
    if ((rc = ps_reserve_all(s, l->stream, s->sbound + std::min(M, D), s->ebound + R))) return rc;
    s->lane = l;  // waited for below, whatever happens
    s->sbound += std::min(M, D);
    s->ebound += R;
    rc = ps_level(l, s, S, d_attr, d_src_off, d_src, R, d_v_off, d_v, M, d_dest_off, d_dest, D,
                  d_next, d_next_off, d_stats);
    std::vector<uint64_t> head(S + 4);
    if (!rc) CK(cudaMemcpyAsync(head.data(), d_stats, (S + 4) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (int wrc = ps_wait(s)) return wrc;
    if (rc || (rc = dgx_lane_sync(l))) return rc;
    const uint64_t NX = head[3 + S];
    if (NX) CK(cudaMemcpyAsync(next, d_next, NX * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    memcpy(next_off, head.data() + 3, (S + 1) * sizeof(uint64_t));
    stats->edges = head[0];
    stats->discovered = head[1];
    stats->to_level = head[2];
    g_stats.d2h += (S + 4 + NX) * sizeof(uint64_t);
    g_stats.uids_out += NX;
    return DGX_OK;
}

extern "C" int dgx_path_result(dgx_path_search* s, uint64_t* uids, uint32_t* attrs, size_t cap, size_t* len) {
    if (!s || !len) return fail(DGX_ERR_ARG, "null argument");
    std::lock_guard<std::mutex> lk(s->mu);
    if (int rc = ps_wait(s)) return rc;
    const uint64_t L = s->st[PS_TO_LEVEL], n = L ? L + 1 : 0;
    *len = n;
    if (n > cap) return fail(DGX_ERR_CAP, "a path of %llu uids does not fit cap %zu", (unsigned long long)n, cap);
    if (n == 0) return DGX_OK;
    if (!uids || !attrs) return fail(DGX_ERR_ARG, "null argument");
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    u64* d_uids;
    u32* d_attrs;
    WsCarve o(l);
    o.plain(&d_uids, n);
    o.plain(&d_attrs, L);
    if (int rc = o.commit()) return rc;
    const uint64_t c = s->st[PS_S_CUR];
    ps_walk_kernel<<<1, 1, 0, l->stream>>>((const u64*)s->sbuf[c], (const u64*)(s->sbuf[c] + 8 * s->scap),
                                           (const u32*)(s->sbuf[c] + 16 * s->scap), (const u64*)s->d_state, L,
                                           d_uids, d_attrs);
    CK(cudaGetLastError());
    count_launches(l, 1);
    CK(cudaMemcpyAsync(uids, d_uids, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(attrs, d_attrs, L * sizeof(uint32_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += n * sizeof(uint64_t) + L * sizeof(uint32_t);
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// Value variables: transformTo over a path and evalLevelAgg's per-row fold (valvar_kernel.cuh)
// ---------------------------------------------------------------------------
constexpr uint64_t kVvMax = uint64_t(1) << 32;  // map sizes, levels, rows, values and dest sizes are 32-bit counts

static uint64_t vv_rtiles(uint64_t n) { return std::max<uint64_t>(1, (n + GB_TILE - 1) / GB_TILE); }

// Radix passes of a level: a dest rank needs bits(ndest - 1), the range two more.
static uint32_t vv_passes(uint64_t ndest) {
    return (gb_bits(ndest ? ndest - 1 : 0) + VV_RANGE_BITS + GB_DIGIT_BITS - 1) / GB_DIGIT_BITS;
}

// One level with device pointers; v_cap bounds v_off[nrows].
struct VvLevel {
    const uint64_t *src, *v_off, *v, *dest;
    uint64_t nrows, v_cap, ndest;
};

// Tickets of a level's scans: two of its own and one per radix pass (at most five passes).
constexpr size_t kVvTickets = 8;

// Every level on the lane, 9 + 3 P launches each (P = vv_passes(ndest)).  Workspace: 80 bytes of words and tickets per
// level and the scans' look-back words, zeroed; 72 bytes per value of the largest v_cap (flag and position 16, keys
// before and after the compaction 16, payloads 8, heads, head indices, segment starts and parts 32) and the largest
// radix hist; both intermediate maps, 16 bytes per entry of the largest intermediate ndest.  The last level
// writes out_key / out_val / *out_len, or only *out_len when the result passes out_cap.
static int vv_run(dgx_lane* l, bool is_float, const uint64_t* d_key, const uint64_t* d_val, uint64_t n,
                  const VvLevel* L, size_t nl, uint64_t* out_key, uint64_t* out_val, uint64_t out_cap,
                  uint64_t* out_len) {
    uint64_t vc = 1, hn = GB_RADIX, mcap = 1, zst = 0;
    for (size_t k = 0; k < nl; ++k) {
        const uint64_t c = std::max<uint64_t>(L[k].v_cap, 1), h = (uint64_t)GB_RADIX * vv_rtiles(c);
        vc = std::max(vc, c);
        hn = std::max(hn, h);
        zst += 2 * scan_tiles(c) + vv_passes(L[k].ndest) * scan_tiles(h);
        if (k + 1 < nl) mcap = std::max<uint64_t>(mcap, L[k].ndest);
    }
    int* bad;
    u64 *level_words, *status, *flag, *pos, *ek[2], *head, *hidx, *sstart, *part, *hist, *hoff, *mk[2], *mv[2];
    u32 *tickets, *ep[2];
    WsCarve ws(l);
    ws.zeroed(&bad, 16);
    ws.zeroed(&level_words, VV_WORDS * nl);
    ws.zeroed(&tickets, kVvTickets * nl);
    ws.zeroed(&status, zst);
    ws.plain(&flag, vc);
    ws.plain(&pos, vc + 1);
    ws.plain(&ek[0], vc);  // compacted keys, and the raw keys (then the sort's spare)
    ws.plain(&ek[1], vc);
    ws.plain(&head, vc);
    ws.plain(&hidx, vc + 1);
    ws.plain(&sstart, vc + 1);
    ws.plain(&part, vc);
    ws.plain(&hist, hn);
    ws.plain(&hoff, hn + 1);
    ws.plain(&mk[0], mcap);
    ws.plain(&mk[1], mcap);
    ws.plain(&mv[0], mcap);
    ws.plain(&mv[1], mcap);
    ws.plain(&ep[0], vc);
    ws.plain(&ep[1], vc);
    if (int rc = ws.commit()) return rc;
    const u64* prev_n = nullptr;
    for (size_t k = 0; k < nl; ++k) {
        const VvLevel& V = L[k];
        const uint64_t c = std::max<uint64_t>(V.v_cap, 1), tv = scan_tiles(c);
        const uint32_t passes = vv_passes(V.ndest);
        u64* words = level_words + VV_WORDS * k;
        u32* ticket = tickets + kVvTickets * k;
        VvParams P{};
        P.first = k == 0;
        P.n0 = n;
        P.mk = k ? mk[(k - 1) & 1] : (const u64*)d_key;
        P.mv = k ? mv[(k - 1) & 1] : (const u64*)d_val;
        P.mn = k ? prev_n : words + VV_W_N0;
        P.src = (const u64*)V.src;
        P.nrows = V.nrows;
        P.v_off = (const u64*)V.v_off;
        P.v = (const u64*)V.v;
        P.v_cap = V.v_cap;
        P.dest = (const u64*)V.dest;
        P.ndest = V.ndest;
        P.is_float = is_float;
        P.tiles = vv_rtiles(c);
        P.words = words;
        P.bad = bad;
        P.err = l->d_err;
        P.flag = flag;
        P.pos = pos;
        P.ek_in = ek[0];
        P.ek_raw = ek[1];
        P.ep_in = ep[0];
        P.ep_raw = ep[1];
        P.head = head;
        P.hidx = hidx;
        P.sstart = sstart;
        P.part = part;
        const bool last = k + 1 == nl;
        P.ok = last ? (u64*)out_key : mk[k & 1];
        P.ov = last ? (u64*)out_val : mv[k & 1];
        P.on = last ? (u64*)out_len : words + VV_W_NX;
        P.o_cap = last ? out_cap : V.ndest;
        prev_n = words + VV_W_NX;
        vv_check_kernel<<<gb_grid(std::max<uint64_t>({V.nrows + 1, V.v_cap, V.ndest, k ? 0 : n})), 256, 0,
                          l->stream>>>(P);
        vv_flags_kernel<<<gb_grid(V.v_cap), 256, 0, l->stream>>>(P);
        scan_u64_kernel<<<(unsigned)tv, EN_NT, 0, l->stream>>>(flag, pos, words + VV_W_M, V.v_cap, status, ticket,
                                                               words + VV_W_E);
        status += tv;
        ticket += 1;
        vv_compact_kernel<<<gb_grid(V.v_cap), 256, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        if (int rc = gb_sort(l, P.tiles, bad, words + VV_W_H, ek, ep, words + VV_W_E, passes, hist, hoff, status,
                             ticket))
            return rc;
        P.ek = ek[passes & 1];
        P.ep = ep[passes & 1];
        vv_heads_kernel<<<gb_grid(V.v_cap), 256, 0, l->stream>>>(P);
        scan_u64_kernel<<<(unsigned)tv, EN_NT, 0, l->stream>>>(head, hidx, words + VV_W_E, V.v_cap, status, ticket,
                                                               words + VV_W_SG);
        status += tv;
        vv_starts_kernel<<<gb_grid(V.v_cap), 256, 0, l->stream>>>(P);
        vv_fold_kernel<<<gb_grid(V.v_cap), 256, 0, l->stream>>>(P);
        vv_combine_kernel<<<gb_grid(V.v_cap), 256, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        count_launches(l, 9);
    }
    return DGX_OK;
}

// The argument checks both forms make before anything is copied.  The host form's v_cap is v_off[nrows].
static int vv_check_type(int type) {
    if (type != DGX_VAL_INT64 && type != DGX_VAL_FLOAT64) return fail(DGX_ERR_ARG, "unknown value type %d", type);
    return DGX_OK;
}

static int vv_check_levels(const VvLevel* L, size_t nl) {
    for (size_t k = 0; k < nl; ++k) {
        const VvLevel& V = L[k];
        if (V.nrows >= kVvMax || V.v_cap >= kVvMax || V.ndest >= kVvMax)
            return fail(DGX_ERR_ARG, "level %zu: rows, values and dest values are 32-bit counts", k);
        if (!V.v_off || (V.nrows && !V.src) || (V.v_cap && !V.v) || (V.ndest && !V.dest))
            return fail(DGX_ERR_ARG, "level %zu: null argument", k);
    }
    return DGX_OK;
}

extern "C" int dgx_dev_var_propagate(dgx_lane* l, int type, const uint64_t* d_key, const uint64_t* d_val, size_t n,
                                     const dgx_var_level* levels, size_t nlevels, uint64_t* d_out_key,
                                     uint64_t* d_out_val, size_t out_cap, uint64_t* d_out_len) {
    if (!l || !levels || !d_out_len || (n && (!d_key || !d_val)) || (out_cap && (!d_out_key || !d_out_val)))
        return fail(DGX_ERR_ARG, "null argument");
    if (int rc = vv_check_type(type)) return rc;
    if (nlevels == 0 || nlevels >= kVvMax || n >= kVvMax)
        return fail(DGX_ERR_ARG, "nlevels of 1 to 2^32 - 1 and a map below 2^32 entries");
    std::vector<VvLevel> L(nlevels);
    for (size_t k = 0; k < nlevels; ++k)
        L[k] = {levels[k].src, levels[k].v_off, levels[k].v, levels[k].dest, levels[k].nrows, levels[k].v_cap,
                levels[k].ndest};
    if (int rc = vv_check_levels(L.data(), nlevels)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_out_len, sizeof(uint64_t));
    if (n == 0) {  // transformTo returns an empty map as it is
        CK(cudaMemsetAsync(d_out_len, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (int rc = vv_run(l, type == DGX_VAL_FLOAT64, d_key, d_val, n, L.data(), nlevels, d_out_key, d_out_val, out_cap,
                        d_out_len))
        return rc;
    g_stats.uids_in += n;
    l->note_output(d_out_key, out_cap * sizeof(uint64_t));
    l->note_output(d_out_val, out_cap * sizeof(uint64_t));
    return DGX_OK;
}

// Copies *d_len entries of the two device arrays to the host when they fit cap: DGX_ERR_CAP with *len set otherwise.
static int vv_finish(dgx_lane* l, const uint64_t* d_len, const uint64_t* d_key, const uint64_t* d_val, uint64_t* key,
                     uint64_t* val, size_t cap, size_t* len) {
    CK(cudaMemcpyAsync(l->h_word, d_len, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (int rc = dgx_lane_sync(l)) return rc;
    const uint64_t G = l->h_word[0];
    *len = G;
    if (G > cap) return fail(DGX_ERR_CAP, "%llu entries do not fit out_cap %zu", (unsigned long long)G, cap);
    if (G) {
        CK(cudaMemcpyAsync(key, d_key, G * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaMemcpyAsync(val, d_val, G * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    }
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += 2 * G * sizeof(uint64_t);
    g_stats.uids_out += G;
    return DGX_OK;
}

extern "C" int dgx_var_propagate(int type, const uint64_t* key, const uint64_t* val, size_t n,
                                 const dgx_var_level* levels, size_t nlevels, uint64_t* out_key, uint64_t* out_val,
                                 size_t out_cap, size_t* out_len) {
    if (!levels || !out_len || (n && (!key || !val)) || (out_cap && (!out_key || !out_val)))
        return fail(DGX_ERR_ARG, "null argument");
    if (int rc = vv_check_type(type)) return rc;
    if (nlevels == 0 || nlevels >= kVvMax || n >= kVvMax)
        return fail(DGX_ERR_ARG, "nlevels of 1 to 2^32 - 1 and a map below 2^32 entries");
    std::vector<VvLevel> L(nlevels);
    for (size_t k = 0; k < nlevels; ++k) {
        const dgx_var_level& V = levels[k];
        if (V.nrows >= kVvMax) return fail(DGX_ERR_ARG, "level %zu: nrows of 2^32 or more", k);
        if (!V.v_off) return fail(DGX_ERR_ARG, "level %zu: null argument", k);
        if (int rc = check_offsets("v_off", V.v_off, V.nrows, kVvMax)) return rc;
        L[k] = {V.src, V.v_off, V.v, V.dest, V.nrows, V.v_off[V.nrows], V.ndest};
    }
    if (int rc = vv_check_levels(L.data(), nlevels)) return rc;
    if (n == 0) {  // transformTo returns an empty map as it is
        *out_len = 0;
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += n;
    uint64_t *d_key, *d_val;  // one copy of each array
    int rc;
    if ((rc = upload_list(l, key, n, &d_key)) || (rc = upload_list(l, val, n, &d_val))) return rc;
    for (size_t k = 0; k < nlevels; ++k) {
        VvLevel& V = L[k];
        uint64_t *s, *o, *v, *d;
        if ((rc = upload_list(l, V.src, V.nrows, &s)) || (rc = upload_list(l, V.v_off, V.nrows + 1, &o)) ||
            (rc = upload_list(l, V.v, V.v_cap, &v)) || (rc = upload_list(l, V.dest, V.ndest, &d)))
            return rc;
        V.src = s;
        V.v_off = o;
        V.v = v;
        V.dest = d;
        g_stats.uids_in += V.nrows + V.v_cap + V.ndest;
    }
    const uint64_t D = L[nlevels - 1].ndest;  // the last map has at most one entry per dest value
    uint64_t *o_len, *o_key, *o_val;
    WsCarve o(l);
    o.plain(&o_len, 1);
    o.plain(&o_key, D);
    o.plain(&o_val, D);
    if ((rc = o.commit())) return rc;
    if ((rc = vv_run(l, type == DGX_VAL_FLOAT64, d_key, d_val, n, L.data(), nlevels, o_key, o_val, D, o_len)))
        return rc;
    return vv_finish(l, o_len, o_key, o_val, out_key, out_val, out_cap, out_len);
}

// 4 launches.  Workspace: 24 bytes per row and the scan's look-back words.
static int la_run(dgx_lane* l, int fn, bool is_float, const uint64_t* d_key, const uint64_t* d_val, uint64_t n,
                  const uint64_t* d_src, uint64_t nrows, const uint64_t* d_v_off, const uint64_t* d_v, uint64_t v_cap,
                  uint64_t* out_key, uint64_t* out_val, uint64_t out_cap, uint64_t* out_len) {
    const uint64_t tr = scan_tiles(nrows);
    VaParams P{};
    u64* status;
    u32* ticket;
    WsCarve ws(l);
    ws.zeroed(&P.bad, 4);
    ws.zeroed(&P.words, VA_WORDS);
    ws.zeroed(&ticket, 8);
    ws.zeroed(&status, tr);
    ws.plain(&P.rval, nrows);
    ws.plain(&P.rflag, nrows);
    ws.plain(&P.rpos, nrows + 1);
    if (int rc = ws.commit()) return rc;
    P.mk = (const u64*)d_key;
    P.mv = (const u64*)d_val;
    P.n = n;
    P.src = (const u64*)d_src;
    P.nrows = nrows;
    P.v_off = (const u64*)d_v_off;
    P.v = (const u64*)d_v;
    P.v_cap = v_cap;
    P.fn = fn;
    P.is_float = is_float;
    P.err = l->d_err;
    P.out_key = (u64*)out_key;
    P.out_val = (u64*)out_val;
    P.out_cap = out_cap;
    P.out_len = (u64*)out_len;
    la_check_kernel<<<gb_grid(std::max<uint64_t>(nrows + 1, n)), 256, 0, l->stream>>>(P);
    la_fold_kernel<<<gb_grid(32 * nrows), 256, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)tr, EN_NT, 0, l->stream>>>(P.rflag, P.rpos, P.words + VA_W_R, nrows, status, ticket,
                                                           P.words + VA_W_G);
    la_write_kernel<<<gb_grid(nrows), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 4);
    return DGX_OK;
}

static int la_check_args(int type, int fn, size_t n, size_t nrows, uint64_t values) {
    if (int rc = vv_check_type(type)) return rc;
    if (fn < DGX_AGG_MIN || fn > DGX_AGG_AVG) return fail(DGX_ERR_ARG, "unknown aggregation %d", fn);
    if (n >= kVvMax || nrows >= kVvMax || values >= kVvMax)
        return fail(DGX_ERR_ARG, "level aggregation sizes are 32-bit: n, nrows and values below 2^32");
    return DGX_OK;
}

extern "C" int dgx_dev_var_level_agg(dgx_lane* l, int type, int fn, const uint64_t* d_key, const uint64_t* d_val,
                                     size_t n, const uint64_t* d_src, size_t nrows, const uint64_t* d_v_off,
                                     const uint64_t* d_v, size_t v_cap, uint64_t* d_out_key, uint64_t* d_out_val,
                                     size_t out_cap, uint64_t* d_out_len) {
    if (!l || !d_out_len || !d_v_off || (n && (!d_key || !d_val)) || (nrows && !d_src) || (v_cap && !d_v) ||
        (out_cap && (!d_out_key || !d_out_val)))
        return fail(DGX_ERR_ARG, "null argument");
    if (int rc = la_check_args(type, fn, n, nrows, v_cap)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_out_len, sizeof(uint64_t));
    if (n == 0 || nrows == 0 || v_cap == 0) {  // no row can hold a value of the map
        CK(cudaMemsetAsync(d_out_len, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (int rc = la_run(l, fn, type == DGX_VAL_FLOAT64, d_key, d_val, n, d_src, nrows, d_v_off, d_v, v_cap, d_out_key,
                        d_out_val, out_cap, d_out_len))
        return rc;
    g_stats.uids_in += n + v_cap;
    l->note_output(d_out_key, out_cap * sizeof(uint64_t));
    l->note_output(d_out_val, out_cap * sizeof(uint64_t));
    return DGX_OK;
}

extern "C" int dgx_var_level_agg(int type, int fn, const uint64_t* key, const uint64_t* val, size_t n,
                                 const uint64_t* src, size_t nrows, const uint64_t* v_off, const uint64_t* v,
                                 uint64_t* out_key, uint64_t* out_val, size_t out_cap, size_t* out_len) {
    if (!out_len || !v_off || (n && (!key || !val)) || (nrows && !src) || (out_cap && (!out_key || !out_val)))
        return fail(DGX_ERR_ARG, "null argument");
    if (int rc = la_check_args(type, fn, n, nrows, 0)) return rc;
    if (int rc = check_offsets("v_off", v_off, nrows, kVvMax)) return rc;
    const uint64_t M = v_off[nrows];
    if (M && !v) return fail(DGX_ERR_ARG, "null argument");
    if (n == 0 || nrows == 0 || M == 0) {  // no row can hold a value of the map
        *out_len = 0;
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += n + nrows + M;
    uint64_t *d_key, *d_val, *d_src, *d_v_off, *d_v;  // one copy of each array
    int rc;
    if ((rc = upload_list(l, key, n, &d_key)) || (rc = upload_list(l, val, n, &d_val)) ||
        (rc = upload_list(l, src, nrows, &d_src)) || (rc = upload_list(l, v_off, nrows + 1, &d_v_off)) ||
        (rc = upload_list(l, v, M, &d_v)))
        return rc;
    uint64_t *o_len, *o_key, *o_val;
    WsCarve o(l);
    o.plain(&o_len, 1);
    o.plain(&o_key, nrows);
    o.plain(&o_val, nrows);
    if ((rc = o.commit())) return rc;
    if ((rc = la_run(l, fn, type == DGX_VAL_FLOAT64, d_key, d_val, n, d_src, nrows, d_v_off, d_v, M, o_key, o_val, nrows,
                     o_len)))
        return rc;
    return vv_finish(l, o_len, o_key, o_val, out_key, out_val, out_cap, out_len);
}

// ---------------------------------------------------------------------------
// math() over value variables: evalMathTree and valueVarAggregation's math branch (math_kernel.cuh)
// ---------------------------------------------------------------------------
static_assert(sizeof(MtProg) == sizeof(dgx_math_node) && offsetof(dgx_math_node, const_word) == offsetof(MtProg, cword),
              "the program is uploaded as it is");

// The program's shape, checked on the host before anything is copied: known ops and constant tags, children earlier in
// post-order and each node but the root the child of exactly one node (Go's tree), leaf indices in range.
static int mt_check_args(const dgx_math_node* prog, size_t nn, const dgx_math_leaf* leaves, size_t nl, size_t nrange,
                         bool device) {
    if (!prog || (nl && !leaves)) return fail(DGX_ERR_ARG, "null argument");
    if (nn == 0 || nn > DGX_MATH_MAX_NODES || nl > DGX_MATH_MAX_LEAVES)
        return fail(DGX_ERR_ARG, "a math program has 1 to %d nodes and at most %d leaves", DGX_MATH_MAX_NODES,
                    DGX_MATH_MAX_LEAVES);
    if (nrange >= kVvMax) return fail(DGX_ERR_ARG, "range of 2^32 uids or more");
    int used[DGX_MATH_MAX_NODES] = {0};
    for (size_t i = 0; i < nn; ++i) {
        const dgx_math_node& g = prog[i];
        if (g.op > DGX_MATH_COND) return fail(DGX_ERR_ARG, "node %zu: unknown op %d", i, g.op);
        if (g.op == DGX_MATH_CONST && g.const_tag != DGX_VAL_INT64 && g.const_tag != DGX_VAL_FLOAT64)
            return fail(DGX_ERR_ARG, "node %zu: a constant is an int64 or a float64", i);
        if (g.op == DGX_MATH_VAR && g.leaf >= nl) return fail(DGX_ERR_ARG, "node %zu: leaf %u of %zu", i, g.leaf, nl);
        for (int c = 0; c < mt_arity(g.op); ++c) {
            if (g.child[c] >= i) return fail(DGX_ERR_ARG, "node %zu: child %u is not earlier in post-order", i, g.child[c]);
            used[g.child[c]] += 1;
        }
    }
    for (size_t i = 0; i + 1 < nn; ++i)
        if (used[i] != 1) return fail(DGX_ERR_ARG, "node %zu is the child of %d nodes: a program is a tree", i, used[i]);
    uint64_t total = 0;
    for (size_t j = 0; j < nl; ++j) {
        const dgx_math_leaf& L = leaves[j];
        if (!L.tag && L.type != DGX_VAL_INT64 && L.type != DGX_VAL_FLOAT64)
            return fail(DGX_ERR_ARG, "leaf %zu: a leaf without tags has type DGX_VAL_INT64 or DGX_VAL_FLOAT64", j);
        if (L.nil && (L.n || L.d_len)) return fail(DGX_ERR_ARG, "leaf %zu: a nil leaf has no entries", j);
        if (!device && L.d_len) return fail(DGX_ERR_ARG, "leaf %zu: d_len belongs to the device form", j);
        if (L.n >= kVvMax) return fail(DGX_ERR_ARG, "leaf %zu: 2^32 entries or more", j);
        if (L.n && (!L.key || !L.word)) return fail(DGX_ERR_ARG, "leaf %zu: null argument", j);
        total += L.n;
    }
    if (total > kMergeMatrixMax) return fail(DGX_ERR_ARG, "the leaves hold 2^32 entries or more");
    return DGX_OK;
}

// 7 launches plus merge_matrix_impl's.  Workspace: the program, leaf table and room offsets copied; counts and words
// zeroed; 42 bytes per unit of the leaves' total room (gathered keys, the union, root tag and word, flag, position)
// plus the merge's own.  Leaves' arrays are device pointers; outputs get *info, and the entries unless refused or past
// out_cap.
static int mt_run(dgx_lane* l, const dgx_math_node* prog, size_t nn, const dgx_math_leaf* leaves, size_t nl,
                  const uint64_t* d_range, size_t nrange, uint64_t* out_key, uint64_t* out_word, uint8_t* out_tag,
                  uint64_t out_cap, uint64_t* info) {
    uint64_t cap = 0;
    for (size_t j = 0; j < nl; ++j) cap += leaves[j].n;
    const uint64_t c1 = std::max<uint64_t>(cap, 1), tiles = scan_tiles(c1);
    MtParams P{};
    MtProg* h_prog;
    MtLeaf* h_leaf;
    u64 *h_cap_off, *status, *ulen;
    u32* ticket;
    WsCarve ws(l);
    ws.copied((MtProg**)&P.prog, &h_prog, nn);
    ws.copied((MtLeaf**)&P.leaf, &h_leaf, std::max<size_t>(nl, 1));
    ws.copied((u64**)&P.cap_off, &h_cap_off, nl + 1);
    ws.zeroed(&P.bad, 4);
    ws.zeroed(&P.words, MT_WORDS);
    ws.zeroed(&P.cnt, nn);
    ws.zeroed(&P.nerr, nn);
    ws.zeroed(&ticket, 4);
    ws.zeroed(&status, tiles);
    ws.plain(&P.plan, nn);
    ws.plain(&P.llen, std::max<size_t>(nl, 1));
    ws.plain(&P.row_off, nl + 1);
    ws.plain(&ulen, 1);
    ws.plain(&P.cat, c1);
    ws.plain((u64**)&P.U, c1);
    ws.plain(&P.rword, c1);
    ws.plain(&P.flag, c1);
    ws.plain(&P.pos, c1 + 1);
    ws.plain(&P.rtag, c1);
    if (int rc = ws.stage()) return rc;
    std::memcpy(h_prog, prog, nn * sizeof(MtProg));
    h_cap_off[0] = 0;
    for (size_t j = 0; j < nl; ++j) {
        const dgx_math_leaf& L = leaves[j];
        h_leaf[j] = MtLeaf{(const u64*)L.key, (const u64*)L.word, L.tag, (const u64*)L.d_len, L.n, L.type, L.nil};
        h_cap_off[j + 1] = h_cap_off[j] + L.n;
    }
    if (int rc = ws.commit()) return rc;
    P.nn = (u32)nn;
    P.nl = (u32)nl;
    P.cap_total = cap;
    P.range = (const u64*)d_range;
    P.nrange = nrange;
    P.ulen = ulen;
    P.err = l->d_err;
    P.out_key = (u64*)out_key;
    P.out_word = (u64*)out_word;
    P.out_tag = out_tag;
    P.out_cap = out_cap;
    P.info = (u64*)info;
    mt_check_kernel<<<gb_grid(cap + (d_range ? nrange : 0)), 256, 0, l->stream>>>(P);
    mt_plan_kernel<<<1, 32, 0, l->stream>>>(P);
    mt_gather_kernel<<<gb_grid(cap), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 3);
    if (int rc = merge_matrix_impl(l, (const uint64_t*)P.cat, (const uint64_t*)P.row_off, nl, cap, (uint64_t*)P.U, c1, (uint64_t*)ulen)) return rc;
    mt_eval_kernel<<<gb_grid(cap), 256, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)tiles, EN_NT, 0, l->stream>>>(P.flag, P.pos, ulen, c1, status, ticket, nullptr);
    mt_finish_kernel<<<1, 32, 0, l->stream>>>(P);
    mt_write_kernel<<<gb_grid(std::max<uint64_t>(cap, d_range ? nrange : 1)), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 4);
    return DGX_OK;
}

extern "C" int dgx_dev_math_eval(dgx_lane* l, const dgx_math_node* prog, size_t nnodes, const dgx_math_leaf* leaves,
                                 size_t nleaves, const uint64_t* d_range, size_t nrange, uint64_t* d_out_key,
                                 uint64_t* d_out_word, uint8_t* d_out_tag, size_t out_cap, uint64_t* d_info) {
    if (!l || !d_info || (out_cap && (!d_out_key || !d_out_word || !d_out_tag)) || (d_range == nullptr && nrange))
        return fail(DGX_ERR_ARG, "null argument");
    if (int rc = mt_check_args(prog, nnodes, leaves, nleaves, nrange, true)) return rc;
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    if (int rc = mt_run(l, prog, nnodes, leaves, nleaves, d_range, nrange, d_out_key, d_out_word, d_out_tag, out_cap,
                        d_info))
        return rc;
    for (size_t j = 0; j < nleaves; ++j) g_stats.uids_in += leaves[j].n;
    l->note_output(d_info, sizeof(uint64_t));
    l->note_output(d_out_key, out_cap * sizeof(uint64_t));
    l->note_output(d_out_word, out_cap * sizeof(uint64_t));
    l->note_output(d_out_tag, out_cap);
    return DGX_OK;
}

extern "C" int dgx_math_eval(const dgx_math_node* prog, size_t nnodes, const dgx_math_leaf* leaves, size_t nleaves,
                             const uint64_t* range, size_t nrange, uint64_t* out_key, uint64_t* out_word,
                             uint8_t* out_tag, size_t out_cap, uint64_t* info) {
    if (!info || (out_cap && (!out_key || !out_word || !out_tag)) || (range == nullptr && nrange))
        return fail(DGX_ERR_ARG, "null argument");
    if (int rc = mt_check_args(prog, nnodes, leaves, nleaves, nrange, false)) return rc;
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    std::vector<dgx_math_leaf> D(leaves, leaves + nleaves);  // one copy of each array
    int rc;
    uint64_t cap = 0;
    for (size_t j = 0; j < nleaves; ++j) {
        dgx_math_leaf& L = D[j];
        uint64_t *k, *w;
        if ((rc = upload_list(l, L.key, L.n, &k)) || (rc = upload_list(l, L.word, L.n, &w))) return rc;
        L.key = k;
        L.word = w;
        if (L.tag) {
            void* t;
            if ((rc = l->ws.alloc(L.n + 1, &t))) return rc;
            if (L.n) CK(cudaMemcpyAsync(t, L.tag, L.n, cudaMemcpyHostToDevice, l->stream));
            g_stats.h2d += L.n;
            L.tag = (const uint8_t*)t;
        }
        g_stats.uids_in += L.n;
        cap += L.n;
    }
    uint64_t* d_range = nullptr;
    if (range && (rc = upload_list(l, range, nrange, &d_range))) return rc;
    const uint64_t R = std::max<uint64_t>(cap + 1, range ? nrange : 1);  // room for any result
    uint64_t *o_info, *o_key, *o_word;
    uint8_t* o_tag;
    WsCarve o(l);
    o.plain(&o_info, 1);
    o.plain(&o_key, R);
    o.plain(&o_word, R);
    o.plain(&o_tag, R);
    if ((rc = o.commit())) return rc;
    if ((rc = mt_run(l, prog, nnodes, D.data(), nleaves, d_range, nrange, o_key, o_word, o_tag, R, o_info))) return rc;
    CK(cudaMemcpyAsync(l->h_word, o_info, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if ((rc = dgx_lane_sync(l))) return rc;
    const uint64_t w = l->h_word[0], G = DGX_MATH_INFO_LEN(w);
    *info = w;
    if (G > out_cap) return fail(DGX_ERR_CAP, "%llu entries do not fit out_cap %zu", (unsigned long long)G, out_cap);
    if (G) {
        CK(cudaMemcpyAsync(out_key, o_key, G * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaMemcpyAsync(out_word, o_word, G * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaMemcpyAsync(out_tag, o_tag, G, cudaMemcpyDeviceToHost, l->stream));
    }
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += G * 17;
    g_stats.uids_out += G;
    return DGX_OK;
}

// ---------------------------------------------------------------------------
// uidsForRegex: a regexp()'s trigram query tree in one call (trigram_kernel.cuh)
// ---------------------------------------------------------------------------
constexpr size_t kTgMaxNodes = size_t(1) << 16, kTgMaxLeaves = size_t(1) << 16, kTgMaxRefs = size_t(1) << 20;
constexpr uint32_t kTgMaxDepth = 32;

// The host plan, from bounds only: the pre-order program, the root's distinct driving leaves and the sum of their
// bounds (dcap, the room of every per-candidate buffer), and whether every node is an OR.
struct TgPlan {
    std::vector<TgOp> prog;
    std::vector<uint32_t> drive;
    uint64_t root_bound = 0, dcap = 0;
    bool all_or = true;
};

struct TgBuild {
    const dgx_query_tree* t;
    const uint64_t* lb;  // leaf bounds
    std::vector<uint64_t> bound;
    std::vector<char> seen;
    TgPlan* P;

    // A node's children as (bound, leaf index or kTgNode | node): its leaves, then its subs, in the given order; an
    // AND's sorted by bound (stably), so that its first child is the smallest, the one that drives it.
    std::vector<std::pair<uint64_t, uint32_t>> children(uint32_t i) const {
        std::vector<std::pair<uint64_t, uint32_t>> ch;
        for (uint32_t k = t->leaf_off[i]; k < t->leaf_off[i + 1]; ++k) ch.push_back({lb[t->leaf_idx[k]], t->leaf_idx[k]});
        for (uint32_t k = t->sub_off[i]; k < t->sub_off[i + 1]; ++k) ch.push_back({bound[t->sub_idx[k]], kTgNode | t->sub_idx[k]});
        if (t->op[i] == DGX_QAND)
            std::stable_sort(ch.begin(), ch.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
        return ch;
    }
    void emit(uint32_t i, uint32_t parent) {
        const uint32_t at = (uint32_t)P->prog.size();
        P->prog.push_back(TgOp{0, parent});
        for (const auto& c : children(i)) {
            if (c.second & kTgNode) emit(c.second & ~kTgNode, at);
            else P->prog.push_back(TgOp{c.second, 0});
        }
        P->prog[at].w0 = kTgNode | (t->op[i] == DGX_QAND ? kTgAnd : 0u) | (uint32_t)P->prog.size();
    }
    void drive(uint32_t i) {
        const auto ch = children(i);
        const size_t n = t->op[i] == DGX_QAND ? 1 : ch.size();
        for (size_t k = 0; k < n; ++k) {
            const uint32_t c = ch[k].second;
            if (c & kTgNode) drive(c & ~kTgNode);
            else if (!seen[c]) {
                seen[c] = 1;
                P->drive.push_back(c);
                P->dcap += lb[c];
            }
        }
    }
};

// The tree's checks and the plan, before anything is copied.  lb[i]: leaf i's bound.
static int tg_plan(const dgx_query_tree* t, const uint64_t* lb, size_t nleaves, TgPlan* P) {
    if (!t) return fail(DGX_ERR_ARG, "null tree");
    const size_t nn = t->nnodes;
    if (nn == 0 || nn >= kTgMaxNodes) return fail(DGX_ERR_ARG, "%zu nodes: between 1 and 2^16 - 1", nn);
    if (!t->op || !t->leaf_off || !t->sub_off) return fail(DGX_ERR_ARG, "null tree array");
    if (t->leaf_off[0] != 0 || t->sub_off[0] != 0) return fail(DGX_ERR_ARG, "leaf_off[0] and sub_off[0] must be 0");
    for (size_t i = 0; i < nn; ++i)
        if (t->leaf_off[i + 1] < t->leaf_off[i] || t->sub_off[i + 1] < t->sub_off[i])
            return fail(DGX_ERR_ARG, "the offsets of node %zu decrease", i);
    if (t->leaf_off[nn] >= kTgMaxRefs) return fail(DGX_ERR_ARG, "%u leaf references: at most 2^20 - 1", t->leaf_off[nn]);
    if ((t->leaf_off[nn] && !t->leaf_idx) || (t->sub_off[nn] && !t->sub_idx)) return fail(DGX_ERR_ARG, "null tree array");
    std::vector<uint32_t> parent(nn, kTgNoParent), depth(nn, 1);
    for (size_t i = 0; i < nn; ++i) {
        const unsigned op = t->op[i];
        if (op != DGX_QAND && op != DGX_QOR) return fail(DGX_ERR_ARG, "node %zu has op %u: not QAnd or QOr", i, op);
        if (op == DGX_QAND && t->leaf_off[i + 1] == t->leaf_off[i] && t->sub_off[i + 1] == t->sub_off[i])
            return fail(DGX_ERR_ARG, "AND node %zu has no trigram and no sub", i);
        if (i > 0 && parent[i] == kTgNoParent) return fail(DGX_ERR_ARG, "node %zu has no parent", i);
        for (uint32_t k = t->leaf_off[i]; k < t->leaf_off[i + 1]; ++k)
            if (t->leaf_idx[k] >= nleaves) return fail(DGX_ERR_ARG, "node %zu names leaf %u of %zu", i, t->leaf_idx[k], nleaves);
        for (uint32_t k = t->sub_off[i]; k < t->sub_off[i + 1]; ++k) {
            const uint32_t s = t->sub_idx[k];
            if (s <= i || s >= nn) return fail(DGX_ERR_ARG, "node %zu names sub %u: subs follow their parent", i, s);
            if (parent[s] != kTgNoParent) return fail(DGX_ERR_ARG, "node %u has two parents", s);
            parent[s] = (uint32_t)i;
            depth[s] = depth[i] + 1;
            if (depth[s] > kTgMaxDepth) return fail(DGX_ERR_ARG, "node %u is deeper than %u", s, kTgMaxDepth);
        }
    }
    TgBuild B{t, lb, std::vector<uint64_t>(nn), std::vector<char>(nleaves, 0), P};
    for (size_t i = nn; i-- > 0;) {  // children have larger indices
        const bool is_and = t->op[i] == DGX_QAND;
        uint64_t b = is_and ? ~uint64_t(0) : 0;
        for (const auto& c : B.children((uint32_t)i)) b = is_and ? std::min(b, c.first) : b + c.first;
        B.bound[i] = b;
        if (is_and) P->all_or = false;
    }
    P->root_bound = B.bound[0];
    if (P->root_bound == 0) return DGX_OK;
    B.emit(0, kTgNoParent);
    B.drive(0);
    return DGX_OK;
}

// The leaves' checks (the layers as for dgx_list_uids_unfiltered_rows, the list offsets, the sum of bounds), then the
// tree's.  rows[i] is pack leaf i.
template <class Row>
static int tg_check(const dgx_query_tree* tree, const Row* rows, size_t npacks, const uint64_t* mut_off,
                    const void* mut_uids, const void* mut_flags, const uint64_t* list_off, size_t nlists, TgPlan* P) {
    const size_t nleaves = npacks + nlists;
    if (nleaves >= kTgMaxLeaves) return fail(DGX_ERR_ARG, "%zu leaves: at most 2^16 - 1", nleaves);
    if ((npacks && (!rows || !mut_off)) || (nlists && !list_off)) return fail(DGX_ERR_ARG, "null argument");
    if (npacks)
        if (int rc = list_unfiltered_check(npacks, mut_off, mut_uids, mut_flags, rows)) return rc;
    if (nlists)
        if (int rc = check_offsets("list_off", list_off, nlists, uint64_t(1) << 32)) return rc;
    std::vector<uint64_t> lb(nleaves);
    uint64_t sum = 0;
    for (size_t i = 0; i < npacks; ++i) sum += lb[i] = exact_len(rows[i]) + (mut_off[i + 1] - mut_off[i]);
    for (size_t j = 0; j < nlists; ++j) sum += lb[npacks + j] = list_off[j + 1] - list_off[j];
    if (sum >> 32) return fail(DGX_ERR_ARG, "the leaves' bounds total %llu: at most 2^32 - 1", (unsigned long long)sum);
    return tg_plan(tree, lb.data(), nleaves, P);
}

// The pipeline of trigram_kernel.cuh for a plan of root bound > 0.  Launches: the unfiltered rows call's 5 when there
// are pack leaves; tg_leaves and tg_gather; merge_matrix_impl's when two or more leaves drive; tg_eval and
// compact_kernel unless every node is an OR.  Workspace: the pack leaves' rows (8 bytes per bound uid plus the rows
// call's 24 per mutable entry and 24 per leaf), the driving rows gathered (8 per dcap), the merge's about 22 per dcap,
// the candidates (8 per dcap) and keep (1 per dcap).  mut_off and list_off are host memory, already checked.
static int trigram_impl(dgx_lane* l, const TgPlan& T, const dgx_dev_pack* const* packs, size_t npacks,
                        const uint64_t* d_mut, const uint8_t* d_flags, const uint64_t* mut_off, const uint64_t* d_lists,
                        const uint64_t* list_off, size_t nlists, uint64_t after, uint64_t* d_out, size_t out_cap,
                        uint64_t* d_out_len) {
    const size_t nleaves = npacks + nlists, nd = T.drive.size();
    const uint64_t dcap = T.dcap;
    uint64_t rows_cap = 0;
    for (size_t i = 0; i < npacks; ++i) rows_cap += exact_len(packs[i]) + (mut_off[i + 1] - mut_off[i]);
    TgParams P;
    TgOp* h_prog;
    uint32_t* h_drive;
    uint64_t* h_loff;
    u64 *row_off, *rows;
    WsCarve ws(l);
    ws.copied(&P.prog, &h_prog, T.prog.size());
    ws.copied(&P.drive, &h_drive, nd);
    ws.copied(&P.list_off, &h_loff, nlists + 1);
    if (int rc = ws.stage()) return rc;
    memcpy(h_prog, T.prog.data(), T.prog.size() * sizeof(TgOp));
    memcpy(h_drive, T.drive.data(), nd * sizeof(uint32_t));
    if (nlists) memcpy(h_loff, list_off, (nlists + 1) * sizeof(uint64_t));
    else h_loff[0] = 0;
    ws.plain(&P.leaf, nleaves);
    ws.plain(&P.drive_off, nd + 1);
    ws.plain(&row_off, npacks + 1);
    ws.plain(&rows, rows_cap + 2);
    if (int rc = ws.commit()) return rc;
    P.npacks = (u32)npacks;
    P.nleaves = (u32)nleaves;
    P.rows = rows;
    P.row_off = row_off;
    P.lists = (const u64*)d_lists;
    P.flags = d_flags;
    P.nmut = npacks ? mut_off[npacks] : 0;
    P.ndrive = (u32)nd;
    P.dcap = dcap;
    P.err = l->d_err;
    int rc;
    if (npacks && (rc = list_unfiltered_impl(l, packs, npacks, d_mut, d_flags, mut_off, after, first_keep(0),
                                             (uint64_t*)rows, rows_cap, (uint64_t*)row_off, nullptr)))
        return rc;
    const bool merge = nd >= 2;
    const bool gather_is_result = T.all_or && !merge;
    if (gather_is_result) {
        P.gathered = (u64*)d_out;
    } else {
        WsCarve g(l);
        g.plain(&P.gathered, dcap + 2);
        if ((rc = g.commit())) return rc;
    }
    P.len_word = gather_is_result ? (u64*)d_out_len : nullptr;
    const unsigned g_val = (unsigned)((dcap + 255) / 256);
    tg_leaves_kernel<<<1, TG_NT, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    tg_gather_kernel<<<g_val, 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 2);
    P.cand = P.gathered;
    P.ncand = P.drive_off + nd;
    if (merge) {
        uint64_t *m_out = d_out, *m_len = d_out_len;
        if (!T.all_or) {
            WsCarve m(l);
            m.plain(&m_len, 8);
            m.plain(&m_out, dcap + 2);
            if ((rc = m.commit())) return rc;
        }
        rc = merge_matrix_impl(l, (const uint64_t*)P.gathered, (const uint64_t*)P.drive_off, nd, dcap, m_out,
                               T.all_or ? out_cap : dcap, m_len);
        if (rc) return rc;
        P.cand = (const u64*)m_out;
        P.ncand = (const u64*)m_len;
    }
    if (!T.all_or) {
        const uint64_t tiles = (dcap + CP_TILE - 1) / CP_TILE;
        CompactParams C;
        WsCarve k(l);
        k.zeroed(&C.status, tiles);
        k.zeroed(&C.ticket, 16);
        k.plain(&P.keep, dcap);
        if ((rc = k.commit())) return rc;
        tg_eval_kernel<<<g_val, 256, 0, l->stream>>>(P);
        CK(cudaGetLastError());
        C.v = P.cand;
        C.keep = P.keep;
        C.m = dcap;
        C.out = (u64*)d_out;
        C.out_cap = out_cap;
        C.out_len = (u64*)d_out_len;
        C.err = l->d_err;
        compact_kernel<<<(unsigned)tiles, CP_NT, 0, l->stream>>>(C);
        CK(cudaGetLastError());
        count_launches(l, 2);
    }
    return DGX_OK;
}

extern "C" int dgx_dev_trigram_query(dgx_lane* l, const dgx_query_tree* tree, const dgx_dev_pack* const* packs,
                                     size_t npacks, const uint64_t* d_mut_uids, const uint8_t* d_mut_flags,
                                     const uint64_t* mut_off, const uint64_t* d_lists, const uint64_t* list_off,
                                     size_t nlists, uint64_t after_uid, uint64_t* d_out, size_t out_cap,
                                     uint64_t* d_out_len) {
    if (!l || !d_out_len) return fail(DGX_ERR_ARG, "null argument");
    TgPlan T;
    if (int rc = tg_check(tree, packs, npacks, mut_off, d_mut_uids, d_mut_flags, list_off, nlists, &T)) return rc;
    if (T.root_bound && (!d_out || (nlists && list_off[nlists] && !d_lists))) return fail(DGX_ERR_ARG, "null argument");
    if (out_cap < T.root_bound)
        return fail(DGX_ERR_CAP, "out_cap (%zu) is below the root's bound (%llu)", out_cap,
                    (unsigned long long)T.root_bound);
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    if (T.root_bound == 0) {
        CK(cudaMemsetAsync(d_out_len, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    const int rc = trigram_impl(l, T, packs, npacks, d_mut_uids, d_mut_flags, mut_off, d_lists, list_off, nlists,
                                after_uid, d_out, out_cap, d_out_len);
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_out_len, sizeof(uint64_t));
    return rc;
}

extern "C" int dgx_trigram_query(const dgx_query_tree* tree, const dgx_pack_ref* refs, size_t npacks,
                                 const uint64_t* mut_uids, const uint8_t* mut_flags, const uint64_t* mut_off,
                                 const uint64_t* lists, const uint64_t* list_off, size_t nlists, uint64_t after_uid,
                                 uint64_t* out, size_t out_cap, size_t* out_len) {
    if (!out_len) return fail(DGX_ERR_ARG, "null out_len");
    TgPlan T;
    if (int rc = tg_check(tree, refs, npacks, mut_off, mut_uids, mut_flags, list_off, nlists, &T)) return rc;
    const uint64_t nmut = npacks ? mut_off[npacks] : 0, nlist = nlists ? list_off[nlists] : 0;
    for (uint64_t k = 0; k < nmut; ++k)
        if (mut_flags[k] & DGX_MUT_VALUE)
            return fail(DGX_ERR_ARG, "mutable entry %llu is not a REF posting", (unsigned long long)k);
    if (T.root_bound && (!out || (nlist && !lists))) return fail(DGX_ERR_ARG, "null argument");
    if (out_cap < T.root_bound)
        return fail(DGX_ERR_CAP, "out_cap (%zu) is below the root's bound (%llu)", out_cap,
                    (unsigned long long)T.root_bound);
    if (T.root_bound == 0) { *out_len = 0; return DGX_OK; }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    PackSet ps(l, refs, npacks);  // nil / empty packs are packs of no blocks
    if (ps.rc) return ps.rc;
    const std::vector<const dgx_dev_pack*> rows = ps.rows();
    uint64_t *d_mut = nullptr, *d_lists;
    const uint8_t* d_flags = nullptr;
    int rc;
    if (npacks && (rc = upload_mut_layers(l, mut_uids, mut_flags, nmut, &d_mut, &d_flags))) return rc;
    if ((rc = upload_list(l, lists, nlist, &d_lists))) return rc;  // the list leaves: one copy
    void* p;
    if ((rc = l->ws.alloc((T.dcap + 10) * sizeof(uint64_t), &p))) return rc;  // the length word, then the values
    uint64_t* d_out = (uint64_t*)p;
    rc = trigram_impl(l, T, rows.data(), npacks, d_mut, d_flags, mut_off, d_lists, list_off, nlists, after_uid,
                      d_out + 8, T.dcap, d_out);
    if (rc) return rc;
    return ps.synced(finish_to_host(l, d_out, d_out + 8, T.dcap, out, out_cap, out_len));
}

// ---------------------------------------------------------------------------
// match(): handleMatchFunction's candidates tested with matchFuzzy against a string value column (match_kernel.cuh)
// ---------------------------------------------------------------------------
constexpr uint64_t kFz32 = uint64_t(1) << 32;     // candidates, column uids, values and bytes are 32-bit counts
constexpr size_t kFzMaxRunes = 64 * FZ_MAX_WORDS;  // the longest query: the long tier holds its words in registers
static_assert(kFzMaxRunes == DGX_MATCH_MAX_RUNES, "include/dgx.h states the query limit");

// utf8.DecodeRuneInString over p[i .. len), as fz_decode on the device.
static uint32_t fz_host_decode(const uint8_t* p, size_t len, size_t i, uint32_t* r) {
    const uint32_t b0 = p[i];
    if (b0 < 0x80) { *r = b0; return 1; }
    *r = FZ_FFFD;
    if (b0 < 0xC2 || b0 > 0xF4) return 1;
    const uint32_t need = b0 < 0xE0 ? 1 : (b0 < 0xF0 ? 2 : 3);
    if (i + need >= len) return 1;
    uint32_t lo = 0x80, hi = 0xBF;
    if (b0 == 0xE0) lo = 0xA0;
    else if (b0 == 0xED) hi = 0x9F;
    else if (b0 == 0xF0) lo = 0x90;
    else if (b0 == 0xF4) hi = 0x8F;
    if (p[i + 1] < lo || p[i + 1] > hi) return 1;
    for (uint32_t k = 2; k <= need; ++k)
        if (p[i + k] < 0x80 || p[i + k] > 0xBF) return 1;
    uint32_t v = b0 & (need == 1 ? 0x1F : need == 2 ? 0x0F : 0x07);
    for (uint32_t k = 1; k <= need; ++k) v = (v << 6) | (p[i + k] & 0x3F);
    *r = v;
    return need + 1;
}

// The query's Peq rows (128 ASCII rows, then one per distinct other rune in ascending order; W words each), from its
// runes as Go's []rune(query) gives them.
struct FzQuery {
    std::vector<uint64_t> peq;
    std::vector<uint32_t> other;
    uint32_t m = 0, W = 1, max = 0;
};

static int fz_query(const uint8_t* q, size_t qlen, int64_t max, FzQuery* Q) {
    if (max < 0 || max > INT32_MAX) return fail(DGX_ERR_ARG, "max is %lld: a non-negative int32", (long long)max);
    if (qlen && !q) return fail(DGX_ERR_ARG, "null query");
    std::vector<uint32_t> runes;
    for (size_t i = 0; i < qlen;) {
        if (runes.size() == kFzMaxRunes) return fail(DGX_ERR_ARG, "the query has more than %zu runes", kFzMaxRunes);
        uint32_t r;
        i += fz_host_decode(q, qlen, i, &r);
        runes.push_back(r);
    }
    Q->m = (uint32_t)runes.size();
    Q->W = std::max<uint32_t>(1, (Q->m + 63) / 64);
    Q->max = (uint32_t)max;
    for (uint32_t r : runes)
        if (r >= 128) Q->other.push_back(r);
    std::sort(Q->other.begin(), Q->other.end());
    Q->other.erase(std::unique(Q->other.begin(), Q->other.end()), Q->other.end());
    Q->peq.assign((128 + Q->other.size()) * Q->W, 0);
    for (uint32_t i = 0; i < Q->m; ++i) {
        const uint32_t r = runes[i];
        const size_t row = r < 128 ? r : 128 + (std::lower_bound(Q->other.begin(), Q->other.end(), r) - Q->other.begin());
        Q->peq[row * Q->W + i / 64] |= uint64_t(1) << (i % 64);
    }
    return DGX_OK;
}

// The column's checks before anything is copied; the host form also checks its offsets (the device form's are checked
// by fz_lookup_kernel).
static int fz_check_column(const dgx_str_column* c, bool host) {
    if (!c) return fail(DGX_ERR_ARG, "null column");
    if (c->n >= kFz32 || c->nvals >= kFz32 || c->nbytes >= kFz32)
        return fail(DGX_ERR_ARG, "column sizes are 32-bit: n %zu, nvals %zu, nbytes %zu", c->n, c->nvals, c->nbytes);
    if (!c->val_off || !c->byte_off || (c->n && !c->uid) || (c->nbytes && !c->bytes))
        return fail(DGX_ERR_ARG, "null column array");
    if (!host) return DGX_OK;
    if (int rc = check_offsets("val_off", c->val_off, c->n, kFz32)) return rc;
    if (c->val_off[c->n] != c->nvals)
        return fail(DGX_ERR_ARG, "val_off[n] is %llu, not nvals (%zu)", (unsigned long long)c->val_off[c->n], c->nvals);
    if (int rc = check_offsets("byte_off", c->byte_off, c->nvals, kFz32)) return rc;
    if (c->byte_off[c->nvals] != c->nbytes)
        return fail(DGX_ERR_ARG, "byte_off[nvals] is %llu, not nbytes (%zu)", (unsigned long long)c->byte_off[c->nvals],
                    c->nbytes);
    return DGX_OK;
}

// uidsForMatch's trigram rows: one OR node over every leaf, planned by the trigram query's checks.
struct FzTree {
    uint8_t op = DGX_QOR;
    uint32_t leaf_off[2] = {0, 0}, sub_off[2] = {0, 0};
    std::vector<uint32_t> leaf_idx;
    dgx_query_tree t{};
    explicit FzTree(size_t nleaves) : leaf_idx(std::max<size_t>(nleaves, 1)) {
        for (size_t i = 0; i < nleaves; ++i) leaf_idx[i] = (uint32_t)i;
        leaf_off[1] = (uint32_t)std::min<size_t>(nleaves, 0xFFFFFFFFu);
        t = dgx_query_tree{1, &op, leaf_off, leaf_idx.data(), sub_off, nullptr};
    }
};

// The test of ccap candidate slots (cand, with the count in the low 32 bits of *cand_len, or ccap when it is null) on
// the lane: 5 launches whatever the candidates, the column, the value lengths and max.  Workspace: Peq, 8 per column
// value (the long-tier queue) and about 33 per candidate slot (value counts, first values, pair offsets, keep flags,
// the look-back words).  col's arrays are device memory.
static int fz_run(dgx_lane* l, const FzQuery& Q, const uint64_t* cand, const uint64_t* cand_len, uint64_t ccap,
                  const dgx_str_column& col, uint64_t* d_out, uint64_t* d_out_len) {
    FzParams P{};
    uint64_t* h_peq;
    uint32_t* h_other;
    u64* status;
    u32* tickets;
    const uint64_t st = scan_tiles(ccap), kt = (ccap + CP_TILE - 1) / CP_TILE;
    WsCarve ws(l);
    ws.copied(&P.peq, &h_peq, Q.peq.size());
    ws.copied(&P.other, &h_other, std::max<size_t>(Q.other.size(), 1));
    if (int rc = ws.stage()) return rc;
    memcpy(h_peq, Q.peq.data(), Q.peq.size() * sizeof(uint64_t));
    h_other[0] = 0;
    if (!Q.other.empty()) memcpy(h_other, Q.other.data(), Q.other.size() * sizeof(uint32_t));
    ws.zeroed(&P.words, 4);
    ws.zeroed(&tickets, 4);
    ws.zeroed(&status, st + kt);
    ws.zeroed(&P.keep, ccap);
    ws.plain(&P.cnt, ccap);
    ws.plain(&P.vlo, ccap);
    ws.plain(&P.pair_off, ccap + 1);
    ws.plain(&P.longq, std::max<size_t>(col.nvals, 1));
    if (int rc = ws.commit()) return rc;
    P.cand = (const u64*)cand;
    P.cand_len = (const u64*)cand_len;
    P.ccap = ccap;
    P.uid = (const u64*)col.uid;
    P.val_off = (const u64*)col.val_off;
    P.byte_off = (const u64*)col.byte_off;
    P.bytes = col.bytes;
    P.n = col.n;
    P.nvals = col.nvals;
    P.nbytes = col.nbytes;
    P.nd = (u32)Q.other.size();
    P.W = Q.W;
    P.m = Q.m;
    P.max = Q.max;
    P.err = l->d_err;
    P.err_bit = kLaneErrMatch;
    fz_lookup_kernel<<<gb_grid(std::max<uint64_t>({ccap, col.n + 1, col.nvals + 1})), 256, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)st, EN_NT, 0, l->stream>>>(P.cnt, P.pair_off, P.words + FZ_W_N, ccap, status, tickets,
                                                            P.words + FZ_W_PAIRS);
    fz_test_kernel<<<gb_grid(col.nvals), 256, 0, l->stream>>>(P);
    fz_long_kernel<<<(unsigned)(2 * g_num_sms), FZ_LONG_NT, 0, l->stream>>>(P);
    CompactParams K;
    K.v = (const u64*)cand;
    K.keep = P.keep;
    K.m = ccap;
    K.out = (u64*)d_out;
    K.out_cap = ccap;
    K.out_len = (u64*)d_out_len;
    K.status = status + st;
    K.ticket = tickets + 1;
    K.err = l->d_err;
    compact_kernel<<<(unsigned)kt, CP_NT, 0, l->stream>>>(K);
    CK(cudaGetLastError());
    count_launches(l, 5);
    return DGX_OK;
}

// The trigram branch's candidates on the lane: the one-OR plan's pipeline into a carved buffer of T.dcap values.
static int fz_trigram_candidates(dgx_lane* l, const TgPlan& T, const dgx_dev_pack* const* packs, size_t npacks,
                                 const uint64_t* d_mut, const uint8_t* d_flags, const uint64_t* mut_off,
                                 const uint64_t* d_lists, const uint64_t* list_off, size_t nlists, uint64_t after,
                                 uint64_t** cand, uint64_t** cand_len) {
    WsCarve c(l);
    c.plain(cand_len, 1);
    c.plain(cand, T.dcap + 2);
    if (int rc = c.commit()) return rc;
    return trigram_impl(l, T, packs, npacks, d_mut, d_flags, mut_off, d_lists, list_off, nlists, after, *cand, T.dcap,
                        *cand_len);
}

// The candidates of a value-column test (match(), regexp()) on the lane, then run(l, cand, cand_len, bound, col, d_out,
// d_out_len), the test's own stages.  The argument checks and refusals are dgx_dev_match's.
template <class Run>
static int str_test_dev(dgx_lane* l, const dgx_dev_pack* const* packs, size_t npacks, const uint64_t* d_mut_uids,
                        const uint8_t* d_mut_flags, const uint64_t* mut_off, const uint64_t* d_lists,
                        const uint64_t* list_off, size_t nlists, uint64_t after_uid, int use_uids,
                        const uint64_t* d_uids, size_t nuids, const uint64_t* d_nuids, const dgx_str_column* col,
                        uint64_t* d_out, size_t out_cap, uint64_t* d_out_len, const Run& run) {
    if (int rc = fz_check_column(col, false)) return rc;
    TgPlan T;
    FzTree tree(npacks + nlists);
    uint64_t bound;
    if (use_uids) {
        if (nuids >= kFz32) return fail(DGX_ERR_ARG, "nuids %zu: at most 2^32 - 1", nuids);
        if (nuids && !d_uids) return fail(DGX_ERR_ARG, "null argument");
        bound = nuids;
    } else {
        if (int rc = tg_check(&tree.t, packs, npacks, mut_off, d_mut_uids, d_mut_flags, list_off, nlists, &T)) return rc;
        if (T.root_bound && nlists && list_off[nlists] && !d_lists) return fail(DGX_ERR_ARG, "null argument");
        bound = T.root_bound;
    }
    if (out_cap < bound)
        return fail(DGX_ERR_CAP, "out_cap (%zu) is below the candidates' bound (%llu)", out_cap,
                    (unsigned long long)bound);
    if (bound && !d_out) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_out_len, sizeof(uint64_t));
    if (bound == 0) {  // no candidate: an empty UidList room, or no trigram row
        CK(cudaMemsetAsync(d_out_len, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    const uint64_t* cand = d_uids;
    const uint64_t* cand_len = d_nuids;
    if (!use_uids) {
        uint64_t *c, *cl;
        if (int rc = fz_trigram_candidates(l, T, packs, npacks, d_mut_uids, d_mut_flags, mut_off, d_lists, list_off,
                                           nlists, after_uid, &c, &cl))
            return rc;
        cand = c;
        cand_len = cl;
    }
    if (int rc = run(l, cand, cand_len, bound, *col, d_out, d_out_len)) return rc;
    g_stats.uids_in += bound;
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    return DGX_OK;
}

// The host form's driver: dgx_match's checks, uploads and branches around run.
template <class Run>
static int str_test_host(const dgx_pack_ref* refs, size_t npacks, const uint64_t* mut_uids, const uint8_t* mut_flags,
                         const uint64_t* mut_off, const uint64_t* lists, const uint64_t* list_off, size_t nlists,
                         uint64_t after_uid, const uint64_t* uids, size_t nuids, const dgx_str_column* col,
                         uint64_t* out, size_t out_cap, size_t* out_len, const Run& run) {
    if (int rc = fz_check_column(col, true)) return rc;
    const bool use_uids = nuids > 0;  // handleMatchFunction / handleRegexFunction: a non-empty UidList is the candidates
    TgPlan T;
    FzTree tree(npacks + nlists);
    uint64_t bound, nmut = 0, nlist = 0;
    if (use_uids) {
        if (nuids >= kFz32) return fail(DGX_ERR_ARG, "nuids %zu: at most 2^32 - 1", nuids);
        if (!uids) return fail(DGX_ERR_ARG, "null argument");
        bound = nuids;
    } else {
        if (int rc = tg_check(&tree.t, refs, npacks, mut_off, mut_uids, mut_flags, list_off, nlists, &T)) return rc;
        nmut = npacks ? mut_off[npacks] : 0;
        nlist = nlists ? list_off[nlists] : 0;
        for (uint64_t k = 0; k < nmut; ++k)
            if (mut_flags[k] & DGX_MUT_VALUE)
                return fail(DGX_ERR_ARG, "mutable entry %llu is not a REF posting", (unsigned long long)k);
        if (T.root_bound && nlist && !lists) return fail(DGX_ERR_ARG, "null argument");
        bound = T.root_bound;
    }
    if (out_cap < bound)
        return fail(DGX_ERR_CAP, "out_cap (%zu) is below the candidates' bound (%llu)", out_cap,
                    (unsigned long long)bound);
    if (bound && !out) return fail(DGX_ERR_ARG, "null argument");
    if (bound == 0) { *out_len = 0; return DGX_OK; }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += bound;
    int rc;
    dgx_str_column D = *col;  // one copy of each column array
    uint64_t *d_uid, *d_voff, *d_boff;
    if ((rc = upload_list(l, col->uid, col->n, &d_uid)) || (rc = upload_list(l, col->val_off, col->n + 1, &d_voff)) ||
        (rc = upload_list(l, col->byte_off, col->nvals + 1, &d_boff)))
        return rc;
    void* b;
    if ((rc = l->ws.alloc(col->nbytes + 16, &b))) return rc;
    if (col->nbytes) CK(cudaMemcpyAsync(b, col->bytes, col->nbytes, cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += col->nbytes;
    D.uid = d_uid;
    D.val_off = d_voff;
    D.byte_off = d_boff;
    D.bytes = (const uint8_t*)b;
    void* p;
    if ((rc = l->ws.alloc((bound + 10) * sizeof(uint64_t), &p))) return rc;  // the length word, then the values
    uint64_t* d_out = (uint64_t*)p;
    if (use_uids) {
        uint64_t* d_uids;
        if ((rc = upload_list(l, uids, nuids, &d_uids))) return rc;
        if ((rc = run(l, d_uids, nullptr, bound, D, d_out + 8, d_out))) return rc;
        if ((rc = finish_to_host(l, d_out, d_out + 8, bound, out, out_cap, out_len))) *out_len = 0;
        return rc;
    }
    PackSet ps(l, refs, npacks);  // nil / empty packs are packs of no blocks
    if (ps.rc) return ps.rc;
    const std::vector<const dgx_dev_pack*> rows = ps.rows();
    uint64_t *d_mut = nullptr, *d_lists, *cand, *cand_len;
    const uint8_t* d_flags = nullptr;
    if (npacks && (rc = upload_mut_layers(l, mut_uids, mut_flags, nmut, &d_mut, &d_flags))) return rc;
    if ((rc = upload_list(l, lists, nlist, &d_lists))) return rc;
    if ((rc = fz_trigram_candidates(l, T, rows.data(), npacks, d_mut, d_flags, mut_off, d_lists, list_off, nlists,
                                    after_uid, &cand, &cand_len)))
        return rc;
    if ((rc = run(l, cand, cand_len, bound, D, d_out + 8, d_out))) return rc;
    if ((rc = ps.synced(finish_to_host(l, d_out, d_out + 8, bound, out, out_cap, out_len)))) *out_len = 0;
    return rc;
}

extern "C" int dgx_dev_match(dgx_lane* l, const dgx_dev_pack* const* packs, size_t npacks, const uint64_t* d_mut_uids,
                             const uint8_t* d_mut_flags, const uint64_t* mut_off, const uint64_t* d_lists,
                             const uint64_t* list_off, size_t nlists, uint64_t after_uid, int use_uids,
                             const uint64_t* d_uids, size_t nuids, const uint64_t* d_nuids, const dgx_str_column* col,
                             const uint8_t* query, size_t query_len, int64_t max, uint64_t* d_out, size_t out_cap,
                             uint64_t* d_out_len) {
    if (!l || !d_out_len) return fail(DGX_ERR_ARG, "null argument");
    FzQuery Q;
    if (int rc = fz_query(query, query_len, max, &Q)) return rc;
    return str_test_dev(l, packs, npacks, d_mut_uids, d_mut_flags, mut_off, d_lists, list_off, nlists, after_uid,
                        use_uids, d_uids, nuids, d_nuids, col, d_out, out_cap, d_out_len,
                        [&](dgx_lane* ln, const uint64_t* c, const uint64_t* cl, uint64_t bound,
                            const dgx_str_column& D, uint64_t* o, uint64_t* ol) {
                            return fz_run(ln, Q, c, cl, bound, D, o, ol);
                        });
}

extern "C" int dgx_match(const dgx_pack_ref* refs, size_t npacks, const uint64_t* mut_uids, const uint8_t* mut_flags,
                         const uint64_t* mut_off, const uint64_t* lists, const uint64_t* list_off, size_t nlists,
                         uint64_t after_uid, const uint64_t* uids, size_t nuids, const dgx_str_column* col,
                         const uint8_t* query, size_t query_len, int64_t max, uint64_t* out, size_t out_cap,
                         size_t* out_len) {
    if (!out_len) return fail(DGX_ERR_ARG, "null out_len");
    FzQuery Q;
    if (int rc = fz_query(query, query_len, max, &Q)) return rc;
    return str_test_host(refs, npacks, mut_uids, mut_flags, mut_off, lists, list_off, nlists, after_uid, uids, nuids,
                         col, out, out_cap, out_len,
                         [&](dgx_lane* ln, const uint64_t* c, const uint64_t* cl, uint64_t bound,
                             const dgx_str_column& D, uint64_t* o, uint64_t* ol) {
                             return fz_run(ln, Q, c, cl, bound, D, o, ol);
                         });
}

// ---------------------------------------------------------------------------
// regexp(): handleRegexFunction's candidates tested with matchRegex against a string value column (regex_kernel.cuh)
// ---------------------------------------------------------------------------
static_assert(rx::kMaxStates == DGX_REGEX_MAX_STATES, "include/dgx.h states the state cap");
static_assert(rx::kTermAbsorb == RX_ABSORB && rx::kTermAccept == RX_ACCEPT && rx::kStartText == RX_START,
              "regex_kernel.cuh reads the compiler's state numbering");

struct dgx_regex_prog {
    rx::Prog p;
};

extern "C" int dgx_regex_compile(const char* pattern, size_t len, int flags, dgx_regex_prog** prog) {
    if (!prog || (len && !pattern)) return fail(DGX_ERR_ARG, "null argument");
    *prog = nullptr;
    if (flags & ~DGX_REGEX_FOLD) return fail(DGX_ERR_ARG, "unknown regex flags %d", flags);
    dgx_regex_prog* r = new dgx_regex_prog;
    const int rc = rx::compile((const uint8_t*)pattern, len, (flags & DGX_REGEX_FOLD) != 0, &r->p);
    if (rc != rx::kOK) delete r;
    if (rc == rx::kRefuse) return fail(DGX_ERR_ARG, "the pattern is outside the compiled subset or invalid");
    if (rc == rx::kTooBig)
        return fail(DGX_ERR_CAP, "the pattern's DFA exceeds %d states (or its byte NFA %d nodes)", rx::kMaxStates,
                    rx::kMaxNfa);
    *prog = r;
    return DGX_OK;
}

extern "C" void dgx_regex_free(dgx_regex_prog* prog) { delete prog; }

extern "C" int dgx_regex_tables(const dgx_regex_prog* prog, size_t* nstates, size_t* nclasses, const uint8_t** cls,
                                const uint16_t** trans, const uint8_t** term) {
    if (!prog || !nstates || !nclasses || !cls || !trans || !term) return fail(DGX_ERR_ARG, "null argument");
    *nstates = prog->p.nstates;
    *nclasses = prog->p.nclasses;
    *cls = prog->p.cls;
    *trans = prog->p.trans.data();
    *term = prog->p.term.data();
    return DGX_OK;
}

// The test of ccap candidate slots on the lane: 5 launches whatever the candidates, the column, the value lengths and
// the program.  Workspace: the program's tables, 8 per column value (the warp tier's queue) and about 33 per candidate
// slot.  col's arrays are device memory.
static int rx_run(dgx_lane* l, const rx::Prog& R, const uint64_t* cand, const uint64_t* cand_len, uint64_t ccap,
                  const dgx_str_column& col, uint64_t* d_out, uint64_t* d_out_len) {
    RxParams P{};
    FzParams& F = P.F;
    unsigned char *h_cls, *h_term;
    uint16_t* h_trans;
    u64* status;
    u32* tickets;
    const uint64_t st = scan_tiles(ccap), kt = (ccap + CP_TILE - 1) / CP_TILE;
    WsCarve ws(l);
    ws.copied(&P.cls, &h_cls, 256);
    ws.copied(&P.trans, &h_trans, R.trans.size());
    ws.copied(&P.term, &h_term, R.term.size());
    if (int rc = ws.stage()) return rc;
    memcpy(h_cls, R.cls, 256);
    memcpy(h_trans, R.trans.data(), R.trans.size() * sizeof(uint16_t));
    memcpy(h_term, R.term.data(), R.term.size());
    ws.zeroed(&F.words, 4);
    ws.zeroed(&tickets, 4);
    ws.zeroed(&status, st + kt);
    ws.zeroed(&F.keep, ccap);
    ws.plain(&F.cnt, ccap);
    ws.plain(&F.vlo, ccap);
    ws.plain(&F.pair_off, ccap + 1);
    ws.plain(&F.longq, std::max<size_t>(col.nvals, 1));
    if (int rc = ws.commit()) return rc;
    F.cand = (const u64*)cand;
    F.cand_len = (const u64*)cand_len;
    F.ccap = ccap;
    F.uid = (const u64*)col.uid;
    F.val_off = (const u64*)col.val_off;
    F.byte_off = (const u64*)col.byte_off;
    F.bytes = col.bytes;
    F.n = col.n;
    F.nvals = col.nvals;
    F.nbytes = col.nbytes;
    F.err = l->d_err;
    F.err_bit = kLaneErrMatch;
    P.nstates = R.nstates;
    P.nclasses = R.nclasses;
    P.warp = R.nstates <= (uint32_t)RX_WARP_STATES;
    const size_t smem = ((size_t)R.nstates * R.nclasses * 2 + 15) / 16 * 16 + 256 + R.nstates;
    const unsigned tgrid = (unsigned)std::min<uint64_t>(gb_grid(col.nvals), 8ull * g_num_sms);
    fz_lookup_kernel<<<gb_grid(std::max<uint64_t>({ccap, col.n + 1, col.nvals + 1})), 256, 0, l->stream>>>(F);
    scan_u64_kernel<<<(unsigned)st, EN_NT, 0, l->stream>>>(F.cnt, F.pair_off, F.words + FZ_W_N, ccap, status, tickets,
                                                            F.words + FZ_W_PAIRS);
    if (R.trans.size() * 2 <= RX_SMEM_TABLE && smem <= 48 * 1024)
        rx_test_kernel<true><<<tgrid, RX_NT, smem, l->stream>>>(P);
    else
        rx_test_kernel<false><<<tgrid, RX_NT, 0, l->stream>>>(P);
    rx_long_kernel<<<(unsigned)(2 * g_num_sms), RX_NT, 0, l->stream>>>(P);
    CompactParams K;
    K.v = (const u64*)cand;
    K.keep = F.keep;
    K.m = ccap;
    K.out = (u64*)d_out;
    K.out_cap = ccap;
    K.out_len = (u64*)d_out_len;
    K.status = status + st;
    K.ticket = tickets + 1;
    K.err = l->d_err;
    compact_kernel<<<(unsigned)kt, CP_NT, 0, l->stream>>>(K);
    CK(cudaGetLastError());
    count_launches(l, 5);
    return DGX_OK;
}

extern "C" int dgx_dev_regex_match(dgx_lane* l, const dgx_dev_pack* const* packs, size_t npacks,
                                   const uint64_t* d_mut_uids, const uint8_t* d_mut_flags, const uint64_t* mut_off,
                                   const uint64_t* d_lists, const uint64_t* list_off, size_t nlists, uint64_t after_uid,
                                   int use_uids, const uint64_t* d_uids, size_t nuids, const uint64_t* d_nuids,
                                   const dgx_str_column* col, const dgx_regex_prog* prog, uint64_t* d_out,
                                   size_t out_cap, uint64_t* d_out_len) {
    if (!l || !d_out_len || !prog) return fail(DGX_ERR_ARG, "null argument");
    return str_test_dev(l, packs, npacks, d_mut_uids, d_mut_flags, mut_off, d_lists, list_off, nlists, after_uid,
                        use_uids, d_uids, nuids, d_nuids, col, d_out, out_cap, d_out_len,
                        [&](dgx_lane* ln, const uint64_t* c, const uint64_t* cl, uint64_t bound,
                            const dgx_str_column& D, uint64_t* o, uint64_t* ol) {
                            return rx_run(ln, prog->p, c, cl, bound, D, o, ol);
                        });
}

extern "C" int dgx_regex_match(const dgx_pack_ref* refs, size_t npacks, const uint64_t* mut_uids,
                               const uint8_t* mut_flags, const uint64_t* mut_off, const uint64_t* lists,
                               const uint64_t* list_off, size_t nlists, uint64_t after_uid, const uint64_t* uids,
                               size_t nuids, const dgx_str_column* col, const dgx_regex_prog* prog, uint64_t* out,
                               size_t out_cap, size_t* out_len) {
    if (!out_len || !prog) return fail(DGX_ERR_ARG, "null argument");
    return str_test_host(refs, npacks, mut_uids, mut_flags, mut_off, lists, list_off, nlists, after_uid, uids, nuids,
                         col, out, out_cap, out_len,
                         [&](dgx_lane* ln, const uint64_t* c, const uint64_t* cl, uint64_t bound,
                             const dgx_str_column& D, uint64_t* o, uint64_t* ol) {
                             return rx_run(ln, prog->p, c, cl, bound, D, o, ol);
                         });
}

// ---------------------------------------------------------------------------
// The compare functions eq / le / lt / ge / gt / between over a typed value column (compare_kernel.cuh)
// ---------------------------------------------------------------------------
static_assert(CMP_LE == DGX_SGF_CMP_LE && CMP_GE == DGX_SGF_CMP_GE && CMP_LT == DGX_SGF_CMP_LT &&
                  CMP_GT == DGX_SGF_CMP_GT && CMP_EQ == DGX_SGF_CMP_EQ && CMP_BETWEEN == DGX_SGF_CMP_BETWEEN,
              "compare_kernel.cuh reads include/dgx.h's op codes");
static_assert(CMP_INT == DGX_VAL_INT64 && CMP_FLOAT == DGX_VAL_FLOAT64 && CMP_BOOL == DGX_VAL_BOOL &&
                  CMP_TIME == DGX_VAL_DATETIME && CMP_STR == DGX_VAL_STRING,
              "compare_kernel.cuh reads include/dgx.h's type codes");
constexpr uint32_t kNsecPerSec = 1000000000u;

// The arguments as the kernels read them: in the caller's order, or (eq on the value path) sorted and deduplicated
// under Equal, NaN dropped and -0 folded to +0.
struct CmpArgs {
    std::vector<uint64_t> word;
    std::vector<uint32_t> nsec;
    std::vector<uint8_t> bytes;
    std::vector<uint64_t> off;  // n + 1 byte offsets (strings)
    size_t n = 0;
};

static int cmp_args(int op, int type, const dgx_val_args* a, bool eq_set, CmpArgs* A) {
    if (op < DGX_SGF_CMP_LE || op > DGX_SGF_CMP_BETWEEN) return fail(DGX_ERR_ARG, "unknown compare op %d", op);
    if (!a) return fail(DGX_ERR_ARG, "null arguments");
    const size_t n = a->n;
    if (n >= kFz32) return fail(DGX_ERR_ARG, "%zu arguments: at most 2^32 - 1", n);
    if (op == DGX_SGF_CMP_BETWEEN && n != 2) return fail(DGX_ERR_ARG, "between takes 2 arguments, not %zu", n);
    if (op == DGX_SGF_CMP_EQ && n < 1) return fail(DGX_ERR_ARG, "eq takes at least 1 argument");
    if (op < DGX_SGF_CMP_EQ && n != 1) return fail(DGX_ERR_ARG, "op %d takes 1 argument, not %zu", op, n);
    std::vector<size_t> idx(n);
    for (size_t k = 0; k < n; ++k) idx[k] = k;
    if (type == DGX_VAL_STRING) {
        if (!a->byte_off) return fail(DGX_ERR_ARG, "null argument byte offsets");
        if (int rc = check_offsets("args byte_off", a->byte_off, n, kFz32)) return rc;
        if (a->byte_off[n] && !a->bytes) return fail(DGX_ERR_ARG, "null argument bytes");
        auto sv = [&](size_t k) {
            return std::string((const char*)a->bytes + a->byte_off[k], (size_t)(a->byte_off[k + 1] - a->byte_off[k]));
        };
        if (eq_set) {
            std::vector<std::string> s(n);
            for (size_t k = 0; k < n; ++k) s[k] = sv(k);
            std::sort(idx.begin(), idx.end(), [&](size_t x, size_t y) { return s[x] < s[y]; });  // bytewise, unsigned
            idx.erase(std::unique(idx.begin(), idx.end(), [&](size_t x, size_t y) { return s[x] == s[y]; }), idx.end());
        }
        A->off.push_back(0);
        for (size_t k : idx) {
            const std::string s = sv(k);
            A->bytes.insert(A->bytes.end(), s.begin(), s.end());
            A->off.push_back(A->bytes.size());
        }
        A->word.assign(idx.size(), 0);
        A->n = idx.size();
        return DGX_OK;
    }
    if (!a->word) return fail(DGX_ERR_ARG, "null argument words");
    if (type == DGX_VAL_DATETIME) {
        if (!a->nsec) return fail(DGX_ERR_ARG, "null argument nanoseconds");
        for (size_t k = 0; k < n; ++k)
            if (a->nsec[k] >= kNsecPerSec) return fail(DGX_ERR_ARG, "argument %zu has %u nanoseconds", k, a->nsec[k]);
    }
    auto key = [&](size_t k) -> uint64_t {  // a total order's key under Equal (NaN dropped before)
        uint64_t w = a->word[k];
        if (type == DGX_VAL_INT64 || type == DGX_VAL_DATETIME) return w ^ (uint64_t(1) << 63);
        if (type == DGX_VAL_BOOL) return w != 0;
        double d;
        memcpy(&d, &w, 8);
        if (d == 0) return uint64_t(1) << 63;  // -0 and +0
        return (w >> 63) ? ~w : w | (uint64_t(1) << 63);
    };
    auto less = [&](size_t x, size_t y) {
        const uint64_t kx = key(x), ky = key(y);
        return kx != ky ? kx < ky : (type == DGX_VAL_DATETIME && a->nsec[x] < a->nsec[y]);
    };
    auto same = [&](size_t x, size_t y) { return !less(x, y) && !less(y, x); };
    if (eq_set) {
        if (type == DGX_VAL_FLOAT64)
            idx.erase(std::remove_if(idx.begin(), idx.end(), [&](size_t k) {
                          double d;
                          memcpy(&d, &a->word[k], 8);
                          return d != d;
                      }), idx.end());
        std::sort(idx.begin(), idx.end(), less);
        idx.erase(std::unique(idx.begin(), idx.end(), same), idx.end());
    }
    for (size_t k : idx) {
        uint64_t w = a->word[k];
        if (eq_set && type == DGX_VAL_FLOAT64 && key(k) == uint64_t(1) << 63) w = 0;  // -0 folded to +0
        if (eq_set && type == DGX_VAL_BOOL) w = w != 0;
        A->word.push_back(w);
        A->nsec.push_back(type == DGX_VAL_DATETIME ? a->nsec[k] : 0);
    }
    A->off.assign(1, 0);
    A->n = idx.size();
    return DGX_OK;
}

// The column's checks before anything is copied; the host form also checks its offsets (the device form's are checked
// by fz_lookup_kernel).  S receives the column as match()'s lookup reads it.
static int cmp_check_column(const dgx_val_column* c, bool host, dgx_str_column* S) {
    if (!c) return fail(DGX_ERR_ARG, "null column");
    const int t = c->type;
    if (t != DGX_VAL_INT64 && t != DGX_VAL_FLOAT64 && t != DGX_VAL_BOOL && t != DGX_VAL_DATETIME && t != DGX_VAL_STRING)
        return fail(DGX_ERR_ARG, "type %d is not compared on the device", t);
    if (t == DGX_VAL_STRING) {
        if (!c->str) return fail(DGX_ERR_ARG, "null string column");
        *S = *c->str;
        return fz_check_column(c->str, host);
    }
    if (c->n >= kFz32 || c->nvals >= kFz32)
        return fail(DGX_ERR_ARG, "column sizes are 32-bit: n %zu, nvals %zu", c->n, c->nvals);
    if (!c->val_off || (c->n && !c->uid) || (c->nvals && !c->word) || (t == DGX_VAL_DATETIME && c->nvals && !c->nsec))
        return fail(DGX_ERR_ARG, "null column array");
    *S = dgx_str_column{c->uid, c->val_off, nullptr, nullptr, c->n, c->nvals, 0};
    if (!host) return DGX_OK;
    if (int rc = check_offsets("val_off", c->val_off, c->n, kFz32)) return rc;
    if (c->val_off[c->n] != c->nvals)
        return fail(DGX_ERR_ARG, "val_off[n] is %llu, not nvals (%zu)", (unsigned long long)c->val_off[c->n], c->nvals);
    return DGX_OK;
}

// The call's parameters common to both paths: the column (device arrays) and the arguments, copied with the workspace.
static void cmp_bind(CmpParams& P, int op, const dgx_val_column& col, const dgx_str_column& S, dgx_lane* l) {
    FzParams& F = P.F;
    F.uid = (const u64*)S.uid;
    F.val_off = (const u64*)S.val_off;
    F.byte_off = (const u64*)S.byte_off;
    F.bytes = S.bytes;
    F.n = S.n;
    F.nvals = S.nvals;
    F.nbytes = S.nbytes;
    F.err = l->d_err;
    F.err_bit = kLaneErrCompare;
    P.type = (u32)col.type;
    P.op = (u32)op;
    P.word = (const u64*)col.word;
    P.nsec = col.nsec;
    P.bad = col.bad;
}
static void cmp_declare_args(WsCarve& ws, CmpParams& P, const CmpArgs& A, uint64_t** hw, uint32_t** hn, uint8_t** hb,
                             uint64_t** ho) {
    ws.copied(&P.aword, hw, std::max<size_t>(A.word.size(), 1));
    ws.copied(&P.ansec, hn, std::max<size_t>(A.nsec.size(), 1));
    ws.copied(&P.aoff, ho, A.off.size());
    ws.copied(&P.abytes, hb, A.bytes.size() + 16);
}
static void cmp_fill_args(CmpParams& P, const CmpArgs& A, uint64_t* hw, uint32_t* hn, uint8_t* hb, uint64_t* ho) {
    hw[0] = 0;
    hn[0] = 0;
    if (!A.word.empty()) memcpy(hw, A.word.data(), A.word.size() * 8);
    if (!A.nsec.empty()) memcpy(hn, A.nsec.data(), A.nsec.size() * 4);
    memcpy(ho, A.off.data(), A.off.size() * 8);
    memset(hb, 0, A.bytes.size() + 16);
    if (!A.bytes.empty()) memcpy(hb, A.bytes.data(), A.bytes.size());
    P.nargs = (u32)A.n;
}

// The value path on the lane for ccap candidate slots: 5 launches whatever the candidates, the column and the
// arguments.  Workspace: the arguments and about 37 bytes per candidate slot (value counts, first values, pair
// offsets, hits, keep flags, the look-back words).
static int cmp_uids_run(dgx_lane* l, int op, const CmpArgs& A, const dgx_val_column& col, const dgx_str_column& S,
                        const uint64_t* cand, const uint64_t* cand_len, uint64_t ccap, uint64_t* d_out,
                        uint64_t* d_out_len, uint32_t* d_counts) {
    CmpParams P{};
    FzParams& F = P.F;
    uint64_t *hw, *ho;
    uint32_t* hn;
    uint8_t* hb;
    u64* status;
    u32* tickets;
    const uint64_t st = scan_tiles(ccap), kt = (ccap + CP_TILE - 1) / CP_TILE;
    WsCarve ws(l);
    cmp_declare_args(ws, P, A, &hw, &hn, &hb, &ho);
    if (int rc = ws.stage()) return rc;
    cmp_fill_args(P, A, hw, hn, hb, ho);
    ws.zeroed(&F.words, 4);
    ws.zeroed(&tickets, 4);
    ws.zeroed(&status, st + kt);
    ws.zeroed(&F.keep, ccap);
    ws.zeroed(&P.hits, ccap);
    ws.plain(&F.cnt, ccap);
    ws.plain(&F.vlo, ccap);
    ws.plain(&F.pair_off, ccap + 1);
    if (int rc = ws.commit()) return rc;
    cmp_bind(P, op, col, S, l);
    F.cand = (const u64*)cand;
    F.cand_len = (const u64*)cand_len;
    F.ccap = ccap;
    P.counts = d_counts;
    const unsigned tgrid = (unsigned)std::min<uint64_t>(gb_grid(S.nvals), 8ull * g_num_sms);
    fz_lookup_kernel<<<gb_grid(std::max<uint64_t>({ccap, S.n + 1, S.nvals + 1})), 256, 0, l->stream>>>(F);
    scan_u64_kernel<<<(unsigned)st, EN_NT, 0, l->stream>>>(F.cnt, F.pair_off, F.words + FZ_W_N, ccap, status, tickets,
                                                            F.words + FZ_W_PAIRS);
    cmp_pairs_kernel<<<tgrid, CMP_NT, 0, l->stream>>>(P);
    cmp_finish_kernel<<<gb_grid(ccap), CMP_NT, 0, l->stream>>>(P);
    CompactParams K;
    K.v = (const u64*)cand;
    K.keep = F.keep;
    K.m = ccap;
    K.out = (u64*)d_out;
    K.out_cap = ccap;
    K.out_len = (u64*)d_out_len;
    K.status = status + st;
    K.ticket = tickets + 1;
    K.err = l->d_err;
    compact_kernel<<<(unsigned)kt, CP_NT, 0, l->stream>>>(K);
    CK(cudaGetLastError());
    count_launches(l, 5);
    return DGX_OK;
}

// The index path on the lane: 4 launches whatever the rows, the column and the arguments.  Workspace: the arguments,
// 4 bytes per row and 16 per value slot (keep flags and their scan).
static int cmp_rows_run(dgx_lane* l, int op, const CmpArgs& A, const dgx_val_column& col, const dgx_str_column& S,
                        const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows, uint64_t v_cap,
                        const uint32_t* row_arg, uint64_t* d_out, uint64_t* d_out_off) {
    CmpParams P{};
    FzParams& F = P.F;
    uint64_t *hw, *ho;
    uint32_t *hn, *hra;
    uint8_t* hb;
    u64* status;
    u32* tickets;
    const uint64_t tiles = scan_tiles(v_cap);
    WsCarve ws(l);
    cmp_declare_args(ws, P, A, &hw, &hn, &hb, &ho);
    ws.copied(&P.row_arg, &hra, nrows);
    if (int rc = ws.stage()) return rc;
    cmp_fill_args(P, A, hw, hn, hb, ho);
    memcpy(hra, row_arg, nrows * sizeof(uint32_t));
    ws.zeroed(&F.words, 4);
    ws.zeroed(&tickets, 2);
    ws.zeroed(&status, tiles);
    ws.plain(&P.flag, std::max<uint64_t>(v_cap, 1));
    ws.plain(&P.pos, v_cap + 1);
    if (int rc = ws.commit()) return rc;
    cmp_bind(P, op, col, S, l);
    F.ccap = 0;  // the lookup checks the column alone
    P.v = (const u64*)d_v;
    P.v_off = (const u64*)d_v_off;
    P.nrows = nrows;
    P.v_cap = v_cap;
    P.out = (u64*)d_out;
    P.out_off = (u64*)d_out_off;
    const uint64_t nt = std::max<uint64_t>(v_cap, nrows + 1);
    fz_lookup_kernel<<<gb_grid(std::max<uint64_t>(S.n + 1, S.nvals + 1)), 256, 0, l->stream>>>(F);
    cmp_rows_kernel<<<gb_grid(nt), CMP_NT, 0, l->stream>>>(P);
    scan_u64_kernel<<<(unsigned)tiles, EN_NT, 0, l->stream>>>(P.flag, P.pos, F.words + CMP_W_M, v_cap, status, tickets,
                                                                nullptr);
    cmp_place_kernel<<<gb_grid(nt), CMP_NT, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 4);
    return DGX_OK;
}

// A host array's device copy in the lane's workspace (nothing for bytes == 0).
static int upload_bytes(dgx_lane* l, const void* h, size_t bytes, void** d) {
    if (int rc = l->ws.alloc(bytes + 16, d)) return rc;
    if (bytes) CK(cudaMemcpyAsync(*d, h, bytes, cudaMemcpyHostToDevice, l->stream));
    g_stats.h2d += bytes;
    return DGX_OK;
}

// The host form's column copy: every array the type needs, with the view match()'s lookup reads.
static int cmp_upload_column(dgx_lane* l, const dgx_val_column* c, dgx_val_column* D, dgx_str_column* S,
                             dgx_str_column* DS) {
    *D = *c;
    const dgx_str_column& H = c->type == DGX_VAL_STRING ? *c->str : *S;
    uint64_t *d_uid, *d_voff;
    int rc;
    if ((rc = upload_list(l, H.uid, H.n, &d_uid)) || (rc = upload_list(l, H.val_off, H.n + 1, &d_voff))) return rc;
    void* p;
    if (c->bad) {
        if ((rc = upload_bytes(l, c->bad, H.nvals, &p))) return rc;
        D->bad = (const uint8_t*)p;
    }
    *DS = H;
    DS->uid = d_uid;
    DS->val_off = d_voff;
    if (c->type == DGX_VAL_STRING) {
        uint64_t* d_boff;
        if ((rc = upload_list(l, H.byte_off, H.nvals + 1, &d_boff))) return rc;
        if ((rc = upload_bytes(l, H.bytes, H.nbytes, &p))) return rc;
        DS->byte_off = d_boff;
        DS->bytes = (const uint8_t*)p;
        return DGX_OK;
    }
    if ((rc = upload_bytes(l, c->word, H.nvals * 8, &p))) return rc;
    D->word = (const uint64_t*)p;
    if (c->type == DGX_VAL_DATETIME) {
        if ((rc = upload_bytes(l, c->nsec, H.nvals * 4, &p))) return rc;
        D->nsec = (const uint32_t*)p;
    }
    return DGX_OK;
}

extern "C" int dgx_dev_compare_uids(dgx_lane* l, int op, const dgx_val_args* args, const dgx_val_column* col,
                                    const uint64_t* d_uids, size_t nuids, const uint64_t* d_nuids, uint64_t* d_out,
                                    size_t out_cap, uint64_t* d_out_len, uint32_t* d_counts) {
    if (!l || !d_out_len) return fail(DGX_ERR_ARG, "null argument");
    dgx_str_column S;
    if (int rc = cmp_check_column(col, false, &S)) return rc;
    CmpArgs A;
    if (int rc = cmp_args(op, col->type, args, op == DGX_SGF_CMP_EQ, &A)) return rc;
    if (nuids >= kFz32) return fail(DGX_ERR_ARG, "nuids %zu: at most 2^32 - 1", nuids);
    if (out_cap < nuids) return fail(DGX_ERR_CAP, "out_cap (%zu) is below nuids (%zu)", out_cap, nuids);
    if (nuids && (!d_uids || !d_out)) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_out_len, sizeof(uint64_t));
    if (nuids == 0) {
        CK(cudaMemsetAsync(d_out_len, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (int rc = cmp_uids_run(l, op, A, *col, S, d_uids, d_nuids, nuids, d_out, d_out_len, d_counts)) return rc;
    g_stats.uids_in += nuids;
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    if (d_counts) l->note_output(d_counts, nuids * sizeof(uint32_t));
    return DGX_OK;
}

extern "C" int dgx_compare_uids(int op, const dgx_val_args* args, const dgx_val_column* col, const uint64_t* uids,
                                size_t nuids, uint64_t* out, size_t out_cap, size_t* out_len, uint32_t* counts) {
    if (!out_len) return fail(DGX_ERR_ARG, "null out_len");
    dgx_str_column S;
    if (int rc = cmp_check_column(col, true, &S)) return rc;
    CmpArgs A;
    if (int rc = cmp_args(op, col->type, args, op == DGX_SGF_CMP_EQ, &A)) return rc;
    if (nuids >= kFz32) return fail(DGX_ERR_ARG, "nuids %zu: at most 2^32 - 1", nuids);
    if (out_cap < nuids) return fail(DGX_ERR_CAP, "out_cap (%zu) is below nuids (%zu)", out_cap, nuids);
    if (nuids && (!uids || !out)) return fail(DGX_ERR_ARG, "null argument");
    if (nuids == 0) { *out_len = 0; return DGX_OK; }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += nuids;
    int rc;
    dgx_val_column D;
    dgx_str_column DS;
    if ((rc = cmp_upload_column(l, col, &D, &S, &DS))) return rc;
    uint64_t* d_uids;
    void* p;
    if ((rc = upload_list(l, uids, nuids, &d_uids))) return rc;
    if ((rc = l->ws.alloc((nuids + 10) * sizeof(uint64_t), &p))) return rc;  // the length word, then the values
    uint64_t* d_out = (uint64_t*)p;
    uint32_t* d_counts = nullptr;
    if (counts && (rc = l->ws.alloc(nuids * sizeof(uint32_t), (void**)&d_counts))) return rc;
    if ((rc = cmp_uids_run(l, op, A, D, DS, d_uids, nullptr, nuids, d_out + 8, d_out, d_counts))) return rc;
    if ((rc = finish_to_host(l, d_out, d_out + 8, nuids, out, out_cap, out_len))) {
        *out_len = 0;
        return rc;
    }
    if (counts) {
        CK(cudaMemcpyAsync(counts, d_counts, nuids * sizeof(uint32_t), cudaMemcpyDeviceToHost, l->stream));
        CK(cudaStreamSynchronize(l->stream));
        g_stats.d2h += nuids * sizeof(uint32_t);
    }
    return DGX_OK;
}

static int cmp_check_row_args(const CmpArgs& A, int op, const uint32_t* row_arg, size_t nrows) {
    if (nrows && !row_arg) return fail(DGX_ERR_ARG, "null row_arg");
    const uint64_t need = op == DGX_SGF_CMP_BETWEEN ? 2 : 1;
    for (size_t r = 0; r < nrows; ++r)
        if (row_arg[r] != CMP_NO_ARG && (uint64_t)row_arg[r] + need > A.n)
            return fail(DGX_ERR_ARG, "row_arg[%zu] is %u: past the %zu arguments", r, row_arg[r], A.n);
    return DGX_OK;
}

extern "C" int dgx_dev_compare_rows(dgx_lane* l, int op, const dgx_val_args* args, const dgx_val_column* col,
                                    const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows, size_t v_cap,
                                    const uint32_t* row_arg, uint64_t* d_out, uint64_t* d_out_off, size_t out_cap) {
    if (!l || !d_out_off) return fail(DGX_ERR_ARG, "null argument");
    dgx_str_column S;
    if (int rc = cmp_check_column(col, false, &S)) return rc;
    CmpArgs A;
    if (int rc = cmp_args(op, col->type, args, false, &A)) return rc;
    if (int rc = cmp_check_row_args(A, op, row_arg, nrows)) return rc;
    if (nrows >= kFz32 || v_cap >= kFz32) return fail(DGX_ERR_ARG, "nrows %zu, v_cap %zu: below 2^32", nrows, v_cap);
    if (out_cap < v_cap) return fail(DGX_ERR_CAP, "out_cap (%zu) is below v_cap (%zu)", out_cap, v_cap);
    if (!d_v_off || (v_cap && (!d_v || !d_out))) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    if (nrows == 0) {
        CK(cudaMemsetAsync(d_out_off, 0, sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (int rc = cmp_rows_run(l, op, A, *col, S, d_v, d_v_off, nrows, v_cap, row_arg, d_out, d_out_off)) return rc;
    g_stats.uids_in += v_cap;
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    return DGX_OK;
}

extern "C" int dgx_compare_rows(int op, const dgx_val_args* args, const dgx_val_column* col, const uint64_t* v,
                                const uint64_t* v_off, size_t nrows, const uint32_t* row_arg, uint64_t* out,
                                uint64_t* out_off, size_t out_cap) {
    if (!out_off || !v_off) return fail(DGX_ERR_ARG, "null argument");
    dgx_str_column S;
    if (int rc = cmp_check_column(col, true, &S)) return rc;
    CmpArgs A;
    if (int rc = cmp_args(op, col->type, args, false, &A)) return rc;
    if (int rc = cmp_check_row_args(A, op, row_arg, nrows)) return rc;
    if (nrows >= kFz32) return fail(DGX_ERR_ARG, "nrows %zu: at most 2^32 - 1", nrows);
    if (int rc = check_offsets("v_off", v_off, nrows, kFz32)) return rc;
    const uint64_t m = v_off[nrows];
    if (out_cap < m) return fail(DGX_ERR_CAP, "out_cap (%zu) is below v_off[nrows] (%llu)", out_cap, (unsigned long long)m);
    if (m && (!v || !out)) return fail(DGX_ERR_ARG, "null argument");
    if (nrows == 0) { out_off[0] = 0; return DGX_OK; }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += m;
    int rc;
    dgx_val_column D;
    dgx_str_column DS;
    if ((rc = cmp_upload_column(l, col, &D, &S, &DS))) return rc;
    uint64_t *d_v, *d_voff, *d_out, *d_off;
    if ((rc = upload_list(l, v, m, &d_v)) || (rc = upload_list(l, v_off, nrows + 1, &d_voff))) return rc;
    if ((rc = l->ws.alloc((m + nrows + 2) * sizeof(uint64_t), (void**)&d_out))) return rc;
    d_off = d_out + m + 1;
    if ((rc = cmp_rows_run(l, op, A, D, DS, d_v, d_voff, nrows, m, row_arg, d_out, d_off))) return rc;
    return batch_to_host(l, d_out, d_off, nrows, out, out_off, out_cap);
}

// ---------------------------------------------------------------------------
// orderasc / orderdesc by a predicate without its index: sortWithoutIndex's value sort over a typed value column,
// nulls last, paged (pred_order_kernel.cuh)
// ---------------------------------------------------------------------------

// The column's checks both forms make before anything is copied: the four sortable types, then compare's checks.
static int po_check_column(const dgx_val_column* c, bool host, dgx_str_column* S) {
    if (!c) return fail(DGX_ERR_ARG, "null column");
    const int t = c->type;
    if (t != DGX_VAL_INT64 && t != DGX_VAL_FLOAT64 && t != DGX_VAL_DATETIME && t != DGX_VAL_STRING)
        return fail(DGX_ERR_ARG, "type %d is not ordered on the device (int64, float64, datetime or string)", t);
    return cmp_check_column(c, host, S);
}

// The datetime key sort's passes: the nanoseconds, then the seconds.
static uint32_t po_key_passes(int type) { return type == DGX_VAL_DATETIME ? PO_NS_PASSES + VO_KEY_PASSES : VO_KEY_PASSES; }

// The whole call on the lane: 38 + 3 P_r launches (51 + 3 P_r for datetime).  Workspace: words, tickets and the
// look-back words, zeroed; per value slot of v_cap about 140 bytes (U and W flags and their scans 32, value index 4,
// N 8, W's uids, words, extras and rows 28, keys 16, radix keys and payloads 24, pair slots 4, the radix hist); per
// row 44; 16 per dest slot.
static int po_run(dgx_lane* l, const dgx_val_column& col, const dgx_str_column& S, int desc, const uint64_t* dest,
                  const uint64_t* dlen, uint64_t dcap, const uint64_t* v, const uint64_t* v_off, uint64_t nrows,
                  uint64_t v_cap, int32_t count, int32_t offset, uint64_t* out, uint64_t* out_off,
                  uint64_t* dest_out, uint64_t* dest_len) {
    const uint64_t vc = std::max<uint64_t>(v_cap, 1), tv = scan_tiles(vc), tr = scan_tiles(nrows), td = scan_tiles(dcap);
    const uint64_t tiles = (vc + GB_TILE - 1) / GB_TILE, hn = (uint64_t)GB_RADIX * tiles, th = scan_tiles(hn);
    const uint32_t pr = vo_row_passes(nrows), kp = po_key_passes(col.type);
    PoParams P{};
    FzParams& F = P.F;
    u64 *status, *ek[2], *hist, *hoff;
    u32 *tickets, *ep[2];
    WsCarve ws(l);
    ws.zeroed(&P.bad, 4);
    ws.zeroed(&P.words, VO_WORDS);
    ws.zeroed(&F.words, 4);
    ws.zeroed(&tickets, 32);
    ws.zeroed(&status, 2 * tv + (kp + pr) * th + tr + td);
    ws.zeroed(&P.rflag, nrows);
    ws.zeroed(&P.mark, dcap);
    ws.plain(&P.uf, vc);
    ws.plain(&P.ux, vc + 1);
    ws.plain(&P.wf, vc);
    ws.plain(&P.wx, vc + 1);
    ws.plain(&P.N, vc);
    ws.plain(&P.wuid, vc);
    ws.plain(&P.wword, vc);
    ws.plain(&P.wext, vc);
    ws.plain(&P.okey, vc);
    ws.plain(&P.okey2, vc);
    ws.plain(&ek[0], vc);
    ws.plain(&ek[1], vc);
    ws.plain(&hist, hn);
    ws.plain(&hoff, hn + 1);
    ws.plain(&P.uoff, nrows + 1);
    ws.plain(&P.woff, nrows + 1);
    ws.plain(&P.plen, nrows);
    ws.plain(&P.po, nrows + 1);
    ws.plain(&P.mx, dcap + 1);
    ws.plain(&P.vj, vc);
    ws.plain(&P.wrow, vc);
    ws.plain(&ep[0], vc);
    ws.plain(&ep[1], vc);
    ws.plain(&P.pairs, vc);
    ws.plain(&P.longrows, nrows);
    ws.plain(&P.pstart, nrows);
    if (int rc = ws.commit()) return rc;
    F.uid = (const u64*)S.uid;
    F.val_off = (const u64*)S.val_off;
    F.byte_off = (const u64*)S.byte_off;
    F.bytes = S.bytes;
    F.n = S.n;
    F.nvals = S.nvals;
    F.nbytes = S.nbytes;
    F.err = l->d_err;
    F.err_bit = kLaneErrPredOrder;
    F.ccap = 0;  // the lookup checks the column alone
    P.type = (u32)col.type;
    P.desc = desc != 0;
    P.word = (const u64*)col.word;
    P.nsec = col.nsec;
    P.vbad = col.bad;
    P.dest = (const u64*)dest;
    P.dlen = (const u64*)dlen;
    P.dcap = dcap;
    P.v = (const u64*)v;
    P.v_off = (const u64*)v_off;
    P.nrows = nrows;
    P.v_cap = v_cap;
    P.count = count;
    P.offset = offset;
    P.tiles = tiles;
    P.err = l->d_err;
    P.ticket = tickets + 31;
    P.ek = ek[0];
    P.ep = ep[0];
    P.out = (u64*)out;
    P.out_off = (u64*)out_off;
    P.dest_out = (u64*)dest_out;
    P.dest_len = (u64*)dest_len;
    u32* ticket = tickets;
    auto scan = [&](const u64* in, u64* o, const u64* n_word, uint64_t n, u64* total) {
        const uint64_t t = scan_tiles(n);
        scan_u64_kernel<<<(unsigned)t, EN_NT, 0, l->stream>>>(in, o, n_word, n, status, ticket, total);
        status += t;
        ticket += 1;
    };
    fz_lookup_kernel<<<gb_grid(std::max<uint64_t>(S.n + 1, S.nvals + 1)), 256, 0, l->stream>>>(F);
    po_check_kernel<<<gb_grid(std::max<uint64_t>({dcap, nrows + 1, v_cap})), 256, 0, l->stream>>>(P);
    po_gather_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P);
    scan(P.uf, P.ux, P.words + VO_W_M, vc, nullptr);
    scan(P.wf, P.wx, P.words + VO_W_M, vc, P.words + VO_W_W);
    po_compact_kernel<<<gb_grid(std::max<uint64_t>(v_cap, nrows + 1)), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 6);
    // W by key (the result is back in buffer c after an even number of passes): a datetime by its nanoseconds, then
    // stably by its seconds; then stably by row
    int c = 0;
    auto sort = [&](uint32_t passes) {
        u64* const k[2] = {ek[c], ek[c ^ 1]};
        u32* const p[2] = {ep[c], ep[c ^ 1]};
        const int rc = gb_sort(l, tiles, P.bad, P.words + VO_W_H, k, p, P.words + VO_W_W, passes, hist, hoff, status,
                               ticket);
        c ^= (int)(passes & 1);
        return rc;
    };
    if (col.type == DGX_VAL_DATETIME) {
        if (int rc = sort(PO_NS_PASSES)) return rc;
        po_rekey_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P, P.okey, ep[c], ek[c ^ 1], ep[c ^ 1]);
        CK(cudaGetLastError());
        count_launches(l, 1);
        c ^= 1;
    }
    if (int rc = sort(VO_KEY_PASSES)) return rc;
    po_rekey_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P, nullptr, ep[c], ek[c ^ 1], ep[c ^ 1]);
    c ^= 1;
    if (int rc = sort(pr)) return rc;
    P.S = ep[c];
    po_tier_kernel<<<gb_grid(v_cap), 256, 0, l->stream>>>(P);
    po_rows_kernel<<<gb_grid(nrows), 256, 0, l->stream>>>(P);
    vo_cta_kernel<<<(unsigned)(2 * g_num_sms), VO_NT, 0, l->stream>>>(P);
    scan(P.plen, P.po, P.words + VO_W_R, nrows, nullptr);
    po_write_kernel<<<gb_grid(std::max<uint64_t>(v_cap, nrows + 1)), 256, 0, l->stream>>>(P);
    scan(P.mark, P.mx, P.words + VO_W_ND, dcap, nullptr);
    vo_dest_kernel<<<gb_grid(dcap), 256, 0, l->stream>>>(P);
    CK(cudaGetLastError());
    count_launches(l, 8);
    return DGX_OK;
}

// The arguments both forms refuse before anything is copied.
static int po_check_args(int32_t count, uint64_t ndest, uint64_t nrows) {
    if (count < 0) return fail(DGX_ERR_ARG, "count %d: processSort refuses a negative count", count);
    if (ndest >= kVoMax || nrows >= kVoMax)
        return fail(DGX_ERR_ARG, "sizes are 32-bit: ndest %llu, nrows %llu", (unsigned long long)ndest,
                    (unsigned long long)nrows);
    return DGX_OK;
}

extern "C" int dgx_dev_pred_order(dgx_lane* l, const dgx_val_column* col, int desc, const uint64_t* d_dest,
                                  size_t ndest, const uint64_t* d_ndest, const uint64_t* d_v, const uint64_t* d_v_off,
                                  size_t nrows, size_t v_cap, int32_t count, int32_t offset, uint64_t* d_out,
                                  uint64_t* d_out_off, size_t out_cap, uint64_t* d_dest_out, size_t dest_cap,
                                  uint64_t* d_dest_len) {
    if (!l || !d_dest_len || !d_v_off || !d_out_off) return fail(DGX_ERR_ARG, "null argument");
    dgx_str_column S;
    if (int rc = po_check_column(col, false, &S)) return rc;
    if (int rc = po_check_args(count, ndest, nrows)) return rc;
    if (v_cap >= kVoMax) return fail(DGX_ERR_ARG, "v_cap %zu: at most 2^32 - 1", v_cap);
    if ((ndest && !d_dest) || (v_cap && !d_v)) return fail(DGX_ERR_ARG, "null argument");
    if (out_cap < v_cap || dest_cap < ndest)
        return fail(DGX_ERR_CAP, "out_cap %zu / dest_cap %zu below the bounds %zu / %zu", out_cap, dest_cap, v_cap,
                    ndest);
    if ((v_cap && !d_out) || (ndest && !d_dest_out)) return fail(DGX_ERR_ARG, "null argument");
    if (int rc = lane_begin_op(l)) return rc;
    g_stats.calls += 1;
    l->note_output(d_dest_len, sizeof(uint64_t));
    l->note_output(d_out_off, (nrows + 1) * sizeof(uint64_t));
    if (ndest == 0 || nrows == 0) {  // no dest value or no row: every row is empty, so is the new dest
        CK(cudaMemsetAsync(d_dest_len, 0, sizeof(uint64_t), l->stream));
        CK(cudaMemsetAsync(d_out_off, 0, (nrows + 1) * sizeof(uint64_t), l->stream));
        return DGX_OK;
    }
    if (int rc = po_run(l, *col, S, desc, d_dest, d_ndest, ndest, d_v, d_v_off, nrows, v_cap, count, offset, d_out,
                        d_out_off, d_dest_out, d_dest_len))
        return rc;
    g_stats.uids_in += ndest + v_cap;
    l->note_output(d_out, out_cap * sizeof(uint64_t));
    l->note_output(d_dest_out, dest_cap * sizeof(uint64_t));
    return DGX_OK;
}

extern "C" int dgx_pred_order(const dgx_val_column* col, int desc, const uint64_t* dest, size_t ndest,
                              const uint64_t* v, const uint64_t* v_off, size_t nrows, int32_t count, int32_t offset,
                              uint64_t* out, uint64_t* out_off, size_t out_cap, uint64_t* dest_out, size_t dest_cap,
                              size_t* dest_len) {
    if (!dest_len || !v_off || !out_off) return fail(DGX_ERR_ARG, "null argument");
    int rc;
    dgx_str_column S;
    if ((rc = po_check_column(col, true, &S))) return rc;
    if ((rc = po_check_args(count, ndest, nrows))) return rc;
    if ((rc = check_offsets("v_off", v_off, nrows, kVoMax))) return rc;
    const uint64_t m = v_off[nrows];
    if ((ndest && !dest) || (m && !v)) return fail(DGX_ERR_ARG, "null argument");
    if (out_cap < m || dest_cap < ndest)
        return fail(DGX_ERR_CAP, "out_cap %zu / dest_cap %zu below the bounds %llu / %zu", out_cap, dest_cap,
                    (unsigned long long)m, ndest);
    if ((m && !out) || (ndest && !dest_out)) return fail(DGX_ERR_ARG, "null argument");
    if (ndest == 0 || nrows == 0) {  // no dest value or no row: every row is empty, so is the new dest
        *dest_len = 0;
        memset(out_off, 0, (nrows + 1) * sizeof(uint64_t));
        return DGX_OK;
    }
    LaneLease lease;
    if (lease.rc) return lease.rc;
    dgx_lane* l = lease.l;
    g_stats.calls += 1;
    g_stats.uids_in += ndest + m;
    dgx_val_column D;
    dgx_str_column DS;
    if ((rc = cmp_upload_column(l, col, &D, &S, &DS))) return rc;
    uint64_t *d_dest, *d_v, *d_v_off;
    if ((rc = upload_list(l, dest, ndest, &d_dest)) || (rc = upload_list(l, v, m, &d_v)) ||
        (rc = upload_list(l, v_off, nrows + 1, &d_v_off)))
        return rc;
    uint64_t *o_len, *o_dest, *o_out, *o_off;
    WsCarve o(l);
    o.plain(&o_len, 1);
    o.plain(&o_dest, ndest);
    o.plain(&o_out, m);
    o.plain(&o_off, nrows + 1);
    if ((rc = o.commit())) return rc;
    if ((rc = po_run(l, D, DS, desc, d_dest, nullptr, ndest, d_v, d_v_off, nrows, m, count, offset, o_out, o_off,
                     o_dest, o_len)))
        return rc;
    CK(cudaMemcpyAsync(l->h_word, o_len, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaMemcpyAsync(l->h_word + 1, o_off + nrows, sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if ((rc = dgx_lane_sync(l))) {
        *dest_len = 0;
        return rc;
    }
    const uint64_t DN = l->h_word[0], K = l->h_word[1];
    *dest_len = DN;
    CK(cudaMemcpyAsync(out_off, o_off, (nrows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (DN) CK(cudaMemcpyAsync(dest_out, o_dest, DN * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    if (K) CK(cudaMemcpyAsync(out, o_out, K * sizeof(uint64_t), cudaMemcpyDeviceToHost, l->stream));
    CK(cudaStreamSynchronize(l->stream));
    g_stats.d2h += (DN + K + nrows + 3) * sizeof(uint64_t);
    g_stats.uids_out += DN + K;
    return DGX_OK;
}

extern "C" uint64_t dgx_merge_matrix_overflows(const dgx_lane* l) { return l ? l->xm_overflows : g_xm_overflows.load(); }
extern "C" uint64_t dgx_filter_tail_queries(const dgx_lane* l) { return l ? l->tail_queries : g_tail_queries.load(); }

// ---------------------------------------------------------------------------
// protobuf wire-format adjacency (host only; see include/dgx.h and wire.hpp)
// ---------------------------------------------------------------------------
extern "C" int dgx_wire_posting_list_pack(const uint8_t* buf, size_t len, const uint8_t** pack, size_t* pack_len) {
    if ((!buf && len) || !pack || !pack_len) return fail(DGX_ERR_ARG, "null argument");
    *pack = nullptr;
    *pack_len = 0;
    wire::Reader r{buf, buf + len};
    uint32_t f, wt;
    bool ok, seen = false;
    while (r.tag(&f, &wt, &ok)) {
        if (f == 1 && wt == 2) {
            // a sub-message split over several occurrences would have to be merged; no encoder emits that
            if (seen) return fail(DGX_ERR_ARG, "pb.PostingList.pack occurs more than once");
            if (!r.bytes(pack, pack_len)) return fail(DGX_ERR_ARG, "truncated pb.PostingList");
            seen = true;
        } else if (!r.skip(wt, f)) {
            return fail(DGX_ERR_ARG, "malformed pb.PostingList");
        }
    }
    if (!ok) return fail(DGX_ERR_ARG, "malformed pb.PostingList");
    return DGX_OK;
}

extern "C" int dgx_wire_pack_measure(const uint8_t* buf, size_t len, size_t* nblocks, size_t* delta_bytes) {
    if ((!buf && len) || !nblocks || !delta_bytes) return fail(DGX_ERR_ARG, "null argument");
    uint32_t bs;
    if (!wire::walk_pack(buf, len, &bs, nblocks, delta_bytes, nullptr)) return fail(DGX_ERR_ARG, "malformed pb.UidPack");
    return DGX_OK;
}

extern "C" int dgx_wire_pack_parse(const uint8_t* buf, size_t len, uint64_t* base, uint32_t* num_uids,
                                   uint64_t* delta_off, uint8_t* deltas, size_t nblocks_cap, size_t delta_cap,
                                   dgx_pack_view* view) {
    if ((!buf && len) || !view || !delta_off) return fail(DGX_ERR_ARG, "null argument");
    uint32_t bs;
    size_t nb, db;
    if (!wire::walk_pack(buf, len, &bs, &nb, &db, nullptr)) return fail(DGX_ERR_ARG, "malformed pb.UidPack");
    if (nb > nblocks_cap || db > delta_cap)
        return fail(DGX_ERR_CAP, "pb.UidPack has %zu blocks / %zu delta bytes, arrays hold %zu / %zu", nb, db, nblocks_cap, delta_cap);
    if ((nb && (!base || !num_uids)) || (db && !deltas)) return fail(DGX_ERR_ARG, "null array");
    const wire::PackArrays a{base, num_uids, delta_off, deltas};
    wire::walk_pack(buf, len, &bs, &nb, &db, &a);
    view->block_size = bs;
    view->nblocks = nb;
    view->base = base;
    view->num_uids = num_uids;
    view->delta_off = delta_off;
    view->deltas = deltas;
    return DGX_OK;
}

extern "C" size_t dgx_wire_list_header(size_t n, uint8_t* hdr) {
    if (n == 0 || !hdr) return 0;
    size_t w = 0;
    hdr[w++] = 0x0A;  // field 1, wire type 2
    uint64_t v = (uint64_t)n * 8u;
    while (v >= 0x80) { hdr[w++] = (uint8_t)(v | 0x80); v >>= 7; }
    hdr[w++] = (uint8_t)v;
    return w;
}

extern "C" int dgx_wire_uid_matrix(const uint64_t* out, const uint64_t* out_off, size_t nrows, uint8_t* buf, size_t buf_cap,
                                   size_t* len) {
    if (!len || (nrows && !out_off)) return fail(DGX_ERR_ARG, "null argument");
    auto varint_len = [](uint64_t v) { size_t n = 1; while (v >= 0x80) { v >>= 7; ++n; } return n; };
    auto put_varint = [](uint8_t* p, uint64_t v) { size_t n = 0; while (v >= 0x80) { p[n++] = (uint8_t)(v | 0x80); v >>= 7; } p[n++] = (uint8_t)v; return n; };
    size_t w = 0;
    for (size_t r = 0; r < nrows; ++r) {
        if (out_off[r + 1] < out_off[r]) return fail(DGX_ERR_ARG, "offsets are not ascending at row %zu", r);
        const uint64_t n = out_off[r + 1] - out_off[r];
        const uint64_t payload = n * 8;
        const uint64_t inner = n ? 1 + varint_len(payload) + payload : 0;  // the row's pb.List message
        const size_t total = 1 + varint_len(inner) + (size_t)inner;
        if (buf) {
            if (w + total > buf_cap) return fail(DGX_ERR_CAP, "uid_matrix does not fit buf_cap (%zu)", buf_cap);
            if (n && !out) return fail(DGX_ERR_ARG, "null values");
            uint8_t* p = buf + w;
            *p++ = 0x0A;
            p += put_varint(p, inner);
            if (n) {
                *p++ = 0x0A;
                p += put_varint(p, payload);
                memcpy(p, out + out_off[r], (size_t)payload);
            }
        }
        w += total;
    }
    *len = w;
    return DGX_OK;
}

extern "C" int dgx_wire_list_decode(const uint8_t* buf, size_t len, uint64_t* out, size_t out_cap, size_t* out_len) {
    if ((!buf && len) || !out_len) return fail(DGX_ERR_ARG, "null argument");
    wire::Reader r{buf, buf + len};
    uint32_t f, wt;
    bool ok;
    size_t n = 0;
    while (r.tag(&f, &wt, &ok)) {
        if (f == 1 && wt == 2) {
            const uint8_t* s;
            size_t nbytes;
            if (!r.bytes(&s, &nbytes) || (nbytes & 7)) return fail(DGX_ERR_ARG, "malformed pb.List");
            const size_t cnt = nbytes / 8;
            if (out) {
                if (n + cnt > out_cap) return fail(DGX_ERR_CAP, "pb.List does not fit out_cap (%zu)", out_cap);
                memcpy(out + n, s, nbytes);  // fixed64 is little-endian on the wire, like the hosts this runs on
            }
            n += cnt;
        } else if (f == 1 && wt == 1) {
            if (r.end - r.p < 8) return fail(DGX_ERR_ARG, "truncated pb.List");
            if (out) {
                if (n + 1 > out_cap) return fail(DGX_ERR_CAP, "pb.List does not fit out_cap (%zu)", out_cap);
                memcpy(out + n, r.p, 8);
            }
            r.p += 8;
            n += 1;
        } else if (!r.skip(wt, f)) {
            return fail(DGX_ERR_ARG, "malformed pb.List");
        }
    }
    if (!ok) return fail(DGX_ERR_ARG, "malformed pb.List");
    *out_len = n;
    return DGX_OK;
}

#ifdef DGX_PIPE_PROF
// Experimental builds only (not part of include/dgx.h): read and clear filter_pipe_kernel's wait counters.
extern "C" int dgx_debug_pprof(uint64_t* out16) {
    unsigned long long h[32];
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpyFromSymbol(h, dgx::g_pprof, sizeof(h)));
    for (int i = 0; i < 32; ++i) out16[i] = h[i];
    memset(h, 0, sizeof(h));
    CK(cudaMemcpyToSymbol(dgx::g_pprof, h, sizeof(h)));
    return DGX_OK;
}
#endif
