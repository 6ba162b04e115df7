// Host orchestration + C ABI of the decoder (include/ruhvro_b200.h).
//
// Replaces the L3 layer of the reference for the direct-decode path:
//   ruhvro/src/deserialize.rs:25-30,53-121 (dispatch, clamp_chunks, build_slices, fan-out)
// with: capacity-planned Arrow arena (sized from what earlier calls on the schema needed) -> ONE fused decode
// kernel (validate, scan, look-back, emit) -> null counts -> one read-back + one stream synchronisation ->
// Arrow C Data Interface export.  A call whose data outgrows the plan (or the first call on a schema) repeats the
// pass once with exact sizes.  Device memory comes from a size-bucketed cache, host output memory from a
// pinned-slab cache; the host path runs chunks on persistent worker threads bound to the GPU's NUMA node.
#include <cuda_runtime.h>
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "../../include/ruhvro_b200.h"
#include "arrow_c.h"
#include "gather.hpp"
#include "ocf.hpp"
#include "jit.hpp"
#include "kernels.cuh"
#include "plan.hpp"
#include "result.hpp"
#include "schema.hpp"

using namespace rv;

// ------------------------------------------------------------------------------------------
// thread-local diagnostics
// ------------------------------------------------------------------------------------------
namespace {

thread_local std::string t_error;
thread_local float t_timings[6] = {0, 0, 0, 0, 0, 0};
thread_local int t_launches = 0;
thread_local const char* t_walker = "none";
thread_local int t_tile = 0;  // rows per tile of the last decode (the smallest, when its chunks ran on several threads)
thread_local long long t_slow_tiles = 0;
thread_local int t_passes = 0;

double env_double(const char* name, double dflt) {
    const char* v = std::getenv(name);
    return v && *v ? std::atof(v) : dflt;
}

rv_status fail(rv_status st, const std::string& msg) {
    t_error = msg;
    return st;
}

#define RV_CUDA(expr)                                                                                  \
    do {                                                                                               \
        cudaError_t e_ = (expr);                                                                       \
        if (e_ != cudaSuccess)                                                                         \
            return fail(RV_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));              \
    } while (0)

// ------------------------------------------------------------------------------------------
// NUMA placement: pinned buffers and the worker threads that fill / drain them belong on the socket the GPU
// hangs off (on the 8-GPU boxes GPUs 0-3 sit on node 0 and 4-7 on node 1; a rank whose pinned memory lives on
// the other socket pays the inter-socket link on every PCIe transfer).  RV_NUMA=0 disables all of it.
// ------------------------------------------------------------------------------------------
struct NumaInfo {
    int node = -1;
    cpu_set_t cpus;
    bool have_cpus = false;
};

bool numa_enabled() {
    static const bool on = [] { const char* e = std::getenv("RV_NUMA"); return !(e && e[0] == '0'); }();
    return on;
}

const NumaInfo& gpu_numa(int device) {
    static std::mutex mu;
    static std::map<int, NumaInfo> cache;
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(device);
    if (it != cache.end()) return it->second;
    NumaInfo info;
    CPU_ZERO(&info.cpus);
    char bus[64] = {0};
    if (numa_enabled() && cudaDeviceGetPCIBusId(bus, int(sizeof bus) - 1, device) == cudaSuccess) {
        for (char* c = bus; *c; ++c) *c = char(std::tolower(static_cast<unsigned char>(*c)));
        const std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
        if (FILE* f = std::fopen(path.c_str(), "r")) {
            int node = -1;
            if (std::fscanf(f, "%d", &node) == 1) info.node = node;
            std::fclose(f);
        }
        if (info.node >= 0) {
            const std::string cl = "/sys/devices/system/node/node" + std::to_string(info.node) + "/cpulist";
            if (FILE* f = std::fopen(cl.c_str(), "r")) {
                char buf[4096] = {0};
                if (std::fgets(buf, sizeof buf, f)) {
                    const char* c = buf;
                    while (*c) {  // "0-31,64-95"
                        char* e = nullptr;
                        long a = std::strtol(c, &e, 10);
                        if (e == c) break;
                        long b = a;
                        if (*e == '-') { c = e + 1; b = std::strtol(c, &e, 10); }
                        for (long x = a; x <= b && x < CPU_SETSIZE; ++x) { CPU_SET(int(x), &info.cpus); info.have_cpus = true; }
                        c = (*e == ',') ? e + 1 : e;
                        if (*e != ',') break;
                    }
                }
                std::fclose(f);
            }
        }
    } else {
        (void)cudaGetLastError();
    }
    return cache[device] = info;
}

// Memory policy of the calling thread: prefer `node` (-1: back to the default policy).  Failures are ignored
// (containers may filter the syscall).
void prefer_node(int node) {
#if defined(SYS_set_mempolicy)
    if (node < 0) { (void)syscall(SYS_set_mempolicy, 0 /*MPOL_DEFAULT*/, nullptr, 0UL); return; }
    unsigned long mask[16] = {0};
    if (node >= int(sizeof mask * 8)) return;
    mask[node / (8 * sizeof(unsigned long))] |= 1UL << (node % (8 * sizeof(unsigned long)));
    (void)syscall(SYS_set_mempolicy, 1 /*MPOL_PREFERRED*/, mask, (unsigned long)(sizeof mask * 8 + 1));
#else
    (void)node;
#endif
}

// Worker threads: run on the GPU's socket (intersected with what the process is allowed to use) and allocate there.
void bind_thread_to_gpu_node(int device) {
    const NumaInfo& ni = gpu_numa(device);
    if (ni.node < 0) return;
    if (ni.have_cpus) {
        cpu_set_t cur, both;
        CPU_ZERO(&cur);
        if (sched_getaffinity(0, sizeof cur, &cur) == 0) {
            CPU_AND(&both, &cur, &ni.cpus);
            if (CPU_COUNT(&both) > 0) (void)sched_setaffinity(0, sizeof both, &both);
        }
    }
    prefer_node(ni.node);
}

// ------------------------------------------------------------------------------------------
// pinned host slabs (cached: cudaHostAlloc of GiB-sized blocks costs hundreds of ms)
// ------------------------------------------------------------------------------------------
class PinnedCache {
  public:
    void* get(size_t bytes, size_t* actual) {
        size_t want = round(bytes);
        {
            std::lock_guard<std::mutex> g(mu_);
            auto it = free_.lower_bound(want);
            if (it != free_.end() && it->first <= want + want / 4 + (1u << 20)) {
                void* p = it->second;
                *actual = it->first;
                cached_ -= it->first;
                free_.erase(it);
                return p;
            }
        }
        // fresh slabs are pinned on the socket of the calling thread's current GPU
        int device = 0, node = -1;
        if (cudaGetDevice(&device) == cudaSuccess) node = gpu_numa(device).node; else (void)cudaGetLastError();
        if (node >= 0) prefer_node(node);
        void* p = nullptr;
        if (cudaHostAlloc(&p, want, cudaHostAllocDefault) != cudaSuccess) {
            (void)cudaGetLastError();
            trim(0);
            if (cudaHostAlloc(&p, want, cudaHostAllocDefault) != cudaSuccess) { (void)cudaGetLastError(); p = nullptr; }
        }
        if (node >= 0) prefer_node(-1);
        if (!p) return nullptr;
        *actual = want;
        return p;
    }
    void put(void* p, size_t actual) {
        if (!p) return;
        {
            std::lock_guard<std::mutex> g(mu_);
            if (cached_ + actual <= kMaxCached) {
                free_.emplace(actual, p);
                cached_ += actual;
                return;
            }
        }
        cudaFreeHost(p);
    }
    void trim(size_t keep) {
        std::lock_guard<std::mutex> g(mu_);
        while (cached_ > keep && !free_.empty()) {
            auto it = std::prev(free_.end());
            cudaFreeHost(it->second);
            cached_ -= it->first;
            free_.erase(it);
        }
    }

  private:
    static constexpr size_t kMaxCached = size_t(24) << 30;
    static size_t round(size_t b) {
        size_t g = b >= (size_t(64) << 20) ? (size_t(16) << 20) : (b >= (1u << 20) ? (1u << 20) : 65536);
        return ((b ? b : 1) + g - 1) / g * g;
    }
    std::mutex mu_;
    std::multimap<size_t, void*> free_;
    size_t cached_ = 0;
};

// ------------------------------------------------------------------------------------------
// device memory: size-bucketed cache over cudaMalloc.  Blocks are only returned once the work that
// used them has been synchronised (every decode path syncs its stream before its buffers die; arenas
// die after their batches are released), so reuse across streams and threads needs no stream ordering.
// ------------------------------------------------------------------------------------------
class DeviceCache {
  public:
    void* get(size_t bytes, int device, size_t* actual) {
        const size_t want = round(bytes);
        {
            std::lock_guard<std::mutex> g(mu_);
            auto& fl = free_[device];
            auto it = fl.lower_bound(want);
            if (it != fl.end() && it->first <= want + want / 4 + (size_t(1) << 20)) {
                void* p = it->second;
                *actual = it->first;
                cached_ -= it->first;
                fl.erase(it);
                return p;
            }
        }
        void* p = nullptr;
        if (cudaMalloc(&p, want) != cudaSuccess) {
            (void)cudaGetLastError();
            trim(device);
            if (cudaMalloc(&p, want) != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
        }
        *actual = want;
        return p;
    }
    void put(void* p, size_t actual, int device) {
        if (!p) return;
        {
            std::lock_guard<std::mutex> g(mu_);
            if (cached_ + actual <= kMaxCached) {
                free_[device].emplace(actual, p);
                cached_ += actual;
                return;
            }
        }
        cudaFree(p);  // the cache is full: give the block back to the driver
    }
    void trim(int device) {
        std::lock_guard<std::mutex> g(mu_);
        auto& fl = free_[device];
        for (auto& kv : fl) { cudaFree(kv.second); cached_ -= kv.first; }
        fl.clear();
    }

  private:
    static constexpr size_t kMaxCached = size_t(40) << 30;  // of the H100's 80 GB
    static size_t round(size_t b) {
        const size_t g = b >= (size_t(32) << 20) ? (size_t(4) << 20) : (b >= (size_t(1) << 20) ? (size_t(256) << 10) : 4096);
        return ((b ? b : 1) + g - 1) / g * g;
    }
    std::mutex mu_;
    std::map<int, std::multimap<size_t, void*>> free_;
    size_t cached_ = 0;
};

DeviceCache& devmem() {
    static DeviceCache* c = new DeviceCache();  // intentionally leaked
    return *c;
}

// Worker streams of the chunk pipeline (created once per device).
cudaStream_t worker_stream(int device, int w) {
    static std::mutex mu;
    static std::map<std::pair<int, int>, cudaStream_t> streams;
    std::lock_guard<std::mutex> g(mu);
    auto key = std::make_pair(device, w);
    auto it = streams.find(key);
    if (it != streams.end()) return it->second;
    cudaStream_t s = nullptr;
    if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) s = nullptr;
    streams[key] = s;
    return s;
}

std::mutex g_host_mu;
std::map<void*, size_t> g_host_sizes;  // rv_host_alloc blocks -> slab size

PinnedCache& pinned() {
    static PinnedCache* c = new PinnedCache();  // intentionally leaked: outlives static destructors
    return *c;
}

// ------------------------------------------------------------------------------------------
// per-process CUDA init
// ------------------------------------------------------------------------------------------
rv_status ensure_cuda(int* device) {
    static std::mutex mu;
    static std::vector<char> inited;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(RV_ERR_CUDA, std::string("no CUDA device available (this library has no CPU fallback): ") + cudaGetErrorString(e));
    RV_CUDA(cudaGetDevice(device));
    std::lock_guard<std::mutex> g(mu);
    if (inited.size() < size_t(n)) inited.resize(size_t(n), 0);
    if (!inited[size_t(*device)]) {
        RV_CUDA(prepare_kernels());
        cudaMemPool_t pool;
        RV_CUDA(cudaDeviceGetDefaultMemPool(&pool, *device));
        unsigned long long thr = ~0ull;  // keep freed blocks in the pool: allocation becomes a free-list pop
        RV_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
        inited[size_t(*device)] = 1;
    }
    return RV_OK;
}

struct DevBuf {  // cached device allocation, returned on scope exit (after the owning stream was synchronised)
    void* p = nullptr;
    size_t actual = 0;
    int device = 0;
    cudaError_t alloc(size_t bytes, cudaStream_t) {
        if (cudaGetDevice(&device) != cudaSuccess) return cudaErrorInvalidDevice;
        p = devmem().get(bytes, device, &actual);
        return p ? cudaSuccess : cudaErrorMemoryAllocation;
    }
    ~DevBuf() { if (p) devmem().put(p, actual, device); }
};

}  // namespace

// ------------------------------------------------------------------------------------------
// schema handle
// ------------------------------------------------------------------------------------------
struct DevicePlan {
    DNode* nodes = nullptr;
    int32_t* sym_off = nullptr;
    uint8_t* sym_bytes = nullptr;
    int16_t* stream_slot = nullptr;
};

// Schema-specialised kernel (NVRTC) of one device: the cubin's architecture and the function attributes are
// per device.
struct JitState {
    bool tried = false;
    bool ok = false;
    std::string status = "not compiled";
    cudaLibrary_t lib = nullptr;
    cudaKernel_t fused = nullptr;
};

// What earlier calls on this schema needed: sizes the output arena and the shared-memory windows of the next call
// without a device round trip.
struct SchemaStats {
    bool valid = false;
    std::vector<double> per_row;   // [S] stream total per record (rows of child spaces / bytes of Utf8 columns)
    double in_per_row = 0;         // input bytes per record
    unsigned long long max_span = 0;   // largest tile input span (bytes)
    unsigned long long max_utf8 = 0;   // largest tile staging need (bytes)
    int tile = 0;                      // the tile (rows) max_span and max_utf8 were measured at
};

// The largest-tile figures of `st` carried over to tiles of `tile` rows.  A tile's bytes are its rows times the mean
// plus an excess; the excess of the largest tile is taken to grow like that of a sum of independent records (with the
// square root of the rows).  An estimate: the first call at the new tile measures it.
static SchemaStats stats_at(const SchemaStats& st, int tile, const Plan& plan) {
    if (!st.valid || st.tile == tile || st.tile == 0) return st;
    SchemaStats o = st;
    o.tile = tile;
    const double g = std::sqrt(double(tile) / double(st.tile));
    auto carry = [&](unsigned long long mx, double per_row, double fixed) -> unsigned long long {
        if (!mx) return 0;
        const double excess = std::max(0.0, double(mx) - (per_row * st.tile + fixed));
        return static_cast<unsigned long long>(std::ceil(per_row * tile + fixed + excess * g));
    };
    double utf8_per_row = 0, n_utf8 = 0;
    for (size_t i = 0; i < plan.streams.size() && i < st.per_row.size(); ++i)
        if (!plan.streams[i].is_rows) { utf8_per_row += st.per_row[i]; n_utf8 += 1; }
    o.max_span = carry(st.max_span, st.in_per_row, 0.0);
    o.max_utf8 = carry(st.max_utf8, utf8_per_row, 31.0 * n_utf8);  // (a tile's staging need has 31 bytes per column of alignment slack)
    return o;
}

struct rv_schema {
    std::atomic<int> refs{1};
    std::shared_ptr<const AvroNode> avro;  // (shared with the handles projected from this one)
    bool supported = false;
    std::string why;              // why it is unsupported / why no plan
    std::vector<ArrowField> fields;  // the columns of the batches, in their order
    bool has_fields = false;
    std::vector<int> keep;        // column projection (rv_schema_project): top-level field of each column; empty: none
    // schema resolution (rv_schema_resolve): `avro` is the writer's schema, `reader` the reader's, `res` pairs them
    std::shared_ptr<const AvroNode> reader;
    std::shared_ptr<const Resolution> res;
    Plan plan;
    bool has_plan = false;
    std::mutex mu;
    std::map<int, DevicePlan> dev;  // device id -> uploaded plan
    std::map<std::pair<int, int>, JitState> jit;    // (device id, tile rows) -> compiled walker
    SchemaStats stats;
};

namespace {

rv_status device_plan(rv_schema* s, int device, DevicePlan* out) {
    std::lock_guard<std::mutex> g(s->mu);
    auto it = s->dev.find(device);
    if (it != s->dev.end()) { *out = it->second; return RV_OK; }
    DevicePlan d;
    const Plan& p = s->plan;
    RV_CUDA(cudaMalloc(&d.nodes, std::max<size_t>(1, p.nodes.size()) * sizeof(DNode)));
    RV_CUDA(cudaMalloc(&d.sym_off, std::max<size_t>(1, p.sym_off.size()) * 4));
    RV_CUDA(cudaMalloc(&d.sym_bytes, std::max<size_t>(1, p.sym_bytes.size())));
    std::vector<int16_t> sslot(std::max<size_t>(1, p.streams.size()), int16_t(-1));
    for (size_t i = 0; i < p.streams.size(); ++i)
        if (!p.streams[i].is_rows) sslot[i] = p.nodes[size_t(p.streams[i].node)].slot_b;
    RV_CUDA(cudaMalloc(&d.stream_slot, sslot.size() * 2));
    RV_CUDA(cudaMemcpy(d.stream_slot, sslot.data(), sslot.size() * 2, cudaMemcpyHostToDevice));
    RV_CUDA(cudaMemcpy(d.nodes, p.nodes.data(), p.nodes.size() * sizeof(DNode), cudaMemcpyHostToDevice));
    if (!p.sym_off.empty()) RV_CUDA(cudaMemcpy(d.sym_off, p.sym_off.data(), p.sym_off.size() * 4, cudaMemcpyHostToDevice));
    if (!p.sym_bytes.empty()) RV_CUDA(cudaMemcpy(d.sym_bytes, p.sym_bytes.data(), p.sym_bytes.size(), cudaMemcpyHostToDevice));
    s->dev[device] = d;
    *out = d;
    return RV_OK;
}

std::atomic<int> g_jit_override{-1};  // -1: follow RV_JIT; 0/1: rv_set_jit_enabled()

bool jit_enabled() {
    const int o = g_jit_override.load(std::memory_order_relaxed);
    if (o >= 0) return o != 0;
    const char* e = std::getenv("RV_JIT");
    return !(e && e[0] == '0');
}

std::string device_arch(int device) {
    if (const char* e = std::getenv("RV_JIT_ARCH")) return e;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return "sm_90a";
    return "sm_" + std::to_string(prop.major) + std::to_string(prop.minor) + ((prop.major >= 9) ? "a" : "");
}

// Compiles + loads the schema-specialised kernel once per (schema, device, tile).  On any failure the generic
// interpreter kernel (also on the GPU) is used and the reason is kept in the state's status.
JitState ensure_jit(rv_schema* s, int device, int tile) {
    if (!jit_enabled()) { JitState d; d.tried = true; d.status = "disabled (RV_JIT=0 / rv_set_jit_enabled(0))"; return d; }
    std::lock_guard<std::mutex> g(s->mu);
    JitState& j = s->jit[{device, tile}];
    if (j.tried) return j;
    j.tried = true;
    const std::string source = generate_kernel_source(s->plan, tile), arch = device_arch(device);
    for (int attempt = 0; attempt < 2; ++attempt) {
        std::vector<char> cubin;
        std::string log;
        if (!jit_cubin(source, arch, &cubin, &log, /*ignore_cache=*/attempt > 0)) { j.status = "NVRTC: " + log; return j; }
        cudaError_t e = cudaLibraryLoadData(&j.lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
        if (e == cudaSuccess) e = cudaLibraryGetKernel(&j.fused, j.lib, "rvj_fused");
        if (e == cudaSuccess) e = cudaFuncSetAttribute(reinterpret_cast<const void*>(j.fused), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        // occupancy is bounded by shared memory: ask for the largest carveout instead of the driver's guess
        if (e == cudaSuccess) e = cudaFuncSetAttribute(reinterpret_cast<const void*>(j.fused), cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        if (e == cudaSuccess) { j.ok = true; j.status = "ok"; return j; }
        // a cached cubin that does not load (corrupt file, other driver) is recompiled once, bypassing the cache
        j.status = std::string("loading the compiled walker failed: ") + cudaGetErrorString(e);
        (void)cudaGetLastError();
        if (j.lib) { cudaLibraryUnload(j.lib); j.lib = nullptr; }
        j.fused = nullptr;
    }
    return j;
}

}  // namespace

// ------------------------------------------------------------------------------------------
// result
// ------------------------------------------------------------------------------------------
namespace {

struct Arena {  // one decode call's output memory; shared by the result and every exported batch
    void* dev = nullptr;
    size_t dev_actual = 0;
    size_t bytes = 0;        // extent of the device arena (capacity-planned layout)
    void* host = nullptr;
    size_t host_actual = 0;
    size_t host_bytes = 0;   // extent of the host slab (exact layout)
    int device = 0;
    void drop_device() {
        if (dev) devmem().put(dev, dev_actual, device);
        dev = nullptr;
    }
    ~Arena() {
        drop_device();
        if (host) pinned().put(host, host_actual);
    }
};

}  // namespace

struct rv_result {
    rv_schema* schema = nullptr;
    std::vector<ChunkOut> chunks;
    std::vector<std::shared_ptr<Arena>> arenas;  // arenas[i] backs chunks[i] (one arena may back many chunks)
    int64_t arrow_bytes = 0;
    ~rv_result() { if (schema) rv_schema_release(schema); }
};

namespace {

// The status of a record's error code (E_ENUM_MAP is an RV_ERR_ENUM with a message of its own).
rv_status status_of(uint32_t code) { return code == E_ENUM_MAP ? RV_ERR_ENUM : rv_status(code); }

const char* err_text(uint32_t code) {
    switch (code) {
        case E_EOF: return "unexpected end of buffer";
        case E_VARINT: return "zigzag varint too long";
        case E_BOOL: return "invalid boolean byte";
        case E_NEG_LEN: return "negative string length";
        case E_BRANCH: return "invalid union branch index";
        case E_ENUM: return "enum index out of range";
        case E_ENUM_MAP: return "enum symbol has neither a reader symbol nor a reader default";
        case E_OVERFLOW: return "Arrow i32 offset overflow (or malformed input offsets)";
        case E_VALUE: return "value does not fit its logical type (uuid text / decimal wider than 128 bits)";
        case E_FRAME: return "framed message: shorter than its header, wrong magic byte or unexpected schema id";
        default: return "decode error";
    }
}

// Small pinned host block per calling thread: the template the device-side call state is initialised from and
// the landing zone of its read-back.
struct HostScratch {
    uint8_t* p = nullptr;
    size_t cap = 0;
    ~HostScratch() { if (p) { cudaFreeHost(p); (void)cudaGetLastError(); } }
    uint8_t* get(size_t bytes) {
        if (bytes > cap) {
            if (p) cudaFreeHost(p);
            p = nullptr;
            cap = 0;
            const size_t want = std::max<size_t>(bytes * 2, 1 << 16);
            if (cudaHostAlloc(reinterpret_cast<void**>(&p), want, cudaHostAllocDefault) != cudaSuccess) { (void)cudaGetLastError(); p = nullptr; return nullptr; }
            cap = want;
        }
        return p;
    }
};
thread_local HostScratch t_scratch;

struct EventPool {  // cudaEventCreate/Destroy per call is measurable at small batch sizes
    cudaEvent_t ev[8] = {};
    int device = -1;
    ~EventPool() { for (auto& e : ev) if (e) cudaEventDestroy(e); (void)cudaGetLastError(); }
    cudaError_t get(int dev, cudaEvent_t** out) {
        if (device != dev) {
            for (auto& e : ev) { if (e) cudaEventDestroy(e); e = nullptr; }
            for (auto& e : ev) { const cudaError_t r = cudaEventCreate(&e); if (r != cudaSuccess) return r; }
            device = dev;
        }
        *out = ev;
        return cudaSuccess;
    }
};
thread_local EventPool t_events;

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Upload of caller memory that is not page-locked (a Rust Vec, a numpy array): cudaMemcpyAsync would stage it inside the
// driver on the calling thread at a fraction of the PCIe rate.  Each thread keeps two pinned pieces instead: the memcpy of
// piece i+1 into one overlaps the DMA of piece i out of the other, and the chunk workers do this side by side.
struct StageRing {
    static constexpr size_t kPiece = size_t(8) << 20;
    uint8_t* buf[2] = {nullptr, nullptr};
    cudaEvent_t done[2] = {nullptr, nullptr};
    int device = -1;
    ~StageRing() { release(); }
    void release() {
        for (int i = 0; i < 2; ++i) {
            if (buf[i]) cudaFreeHost(buf[i]);
            if (done[i]) cudaEventDestroy(done[i]);
            buf[i] = nullptr; done[i] = nullptr;
        }
        (void)cudaGetLastError();
        device = -1;
    }
    bool ready(int dev) {
        if (device == dev) return true;
        release();
        for (int i = 0; i < 2; ++i) {
            if (cudaHostAlloc(reinterpret_cast<void**>(&buf[i]), kPiece, cudaHostAllocDefault) != cudaSuccess ||
                cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming) != cudaSuccess) { release(); return false; }
        }
        device = dev;
        return true;
    }
    // dst[0, bytes) <- src, in order on `stream`.  The pieces are free again when the stream has drained.
    cudaError_t upload(uint8_t* dst, const uint8_t* src, size_t bytes, cudaStream_t stream) {
        int slot = 0;
        for (size_t o = 0; o < bytes; o += kPiece, slot ^= 1) {
            const size_t len = std::min(kPiece, bytes - o);
            cudaError_t e = cudaEventSynchronize(done[slot]);  // the DMA that last read this piece (no-op the first time)
            if (e != cudaSuccess) return e;
            std::memcpy(buf[slot], src + o, len);
            e = cudaMemcpyAsync(dst + o, buf[slot], len, cudaMemcpyHostToDevice, stream);
            if (e == cudaSuccess) e = cudaEventRecord(done[slot], stream);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
};
thread_local StageRing t_stage;

// true when `p` is ordinary pageable host memory (not pinned, registered, managed or device memory)
bool is_pageable(const void* p) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { (void)cudaGetLastError(); return true; }
    return at.type == cudaMemoryTypeUnregistered;
}

// Host -> device on `stream`: through the calling thread's staging ring when the source is pageable and big enough to care.
cudaError_t upload(uint8_t* dst, const uint8_t* src, size_t bytes, int device, cudaStream_t stream) {
    if (bytes >= (size_t(1) << 20) && is_pageable(src) && t_stage.ready(device)) return t_stage.upload(dst, src, bytes, stream);
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream);
}


// Error paths return cached device blocks (DevBuf) while work may still be queued on the stream: drain it first.
struct SyncOnExit {
    cudaStream_t stream;
    bool armed = true;
    ~SyncOnExit() { if (armed) { cudaStreamSynchronize(stream); (void)cudaGetLastError(); } }
};

// Hints of the host path, which can read the offsets: exact input bytes and the largest tile span.
struct InputHints {
    int64_t total_bytes = -1;
    const int64_t* offsets = nullptr;  // the call's n + 1 offsets in host memory
    rv_framing framing = {0, 0, -1};   // framed input (rv_decode_*_framed)
};

// The largest input span of a tile of `tile` rows (tiles count from each chunk's first row, as tile_of does).
int64_t max_tile_span(const int64_t* offsets, int64_t n, int64_t k, int tile) {
    const int64_t cr = n / k;
    int64_t mx = 0;
    for (int64_t j = 0; j < k; ++j) {
        const int64_t cs = j * cr, ce = (j == k - 1) ? n : cs + cr;
        for (int64_t a = cs; a < ce; a += tile) mx = std::max(mx, offsets[std::min(a + tile, ce)] - offsets[a]);
    }
    return mx;
}

// ---- the decode call ------------------------------------------------------------------------
rv_status decode_on_device(rv_schema* s, const uint8_t* d_data, const int64_t* d_offsets, int64_t n, int64_t num_chunks,
                           const InputHints& hints, cudaStream_t stream, int device, rv_result** out, int64_t record_base = 0) {
    const Plan& plan = s->plan;
    const int S = int(plan.streams.size());
    const int Sx = std::max(S, 1);
    const int n_slots = int(plan.slots.size());
    // clamp_chunks (deserialize.rs:53-55)
    int64_t k64 = clamp_chunks(num_chunks, n);
    if (k64 > (int64_t(1) << 24)) return fail(RV_ERR_INVALID, "num_chunks above 2^24 is not supported");
    const int k = int(k64);
    const int64_t chunk_rows = n / k;  // build_slices (:57-68)
    const int64_t last_rows = n - chunk_rows * (k - 1);

    auto res = std::make_unique<rv_result>();
    res->schema = rv_schema_retain(s);
    auto arena_sp = std::make_shared<Arena>();
    arena_sp->device = device;

    for (int i = 0; i < 4; ++i) t_timings[i] = 0;
    t_launches = 0;
    t_passes = 0;
    // RV_TRACE=1: host-side phase times of this call on stderr (development aid)
    static const bool trace = std::getenv("RV_TRACE") && std::getenv("RV_TRACE")[0] == '1';
    auto t_prev = std::chrono::steady_clock::now();
    std::string trace_line;
    auto mark = [&](const char* what) {
        if (!trace) return;
        const auto now = std::chrono::steady_clock::now();
        trace_line += std::string(what) + "=" + std::to_string(std::chrono::duration<double, std::micro>(now - t_prev).count()).substr(0, 6) + "us ";
        t_prev = now;
    };

    std::vector<unsigned long long> chunk_tot(size_t(k) * size_t(Sx), 0ull);

    if (n == 0) {  // one empty batch; offsets buffers hold the single 0 entry
        Layout L = compute_layout(plan, 0, k, chunk_tot.data());
        res->chunks = std::move(L.chunks);
        arena_sp->bytes = L.total_bytes;
        arena_sp->dev = devmem().get(std::max<size_t>(L.total_bytes, 64), device, &arena_sp->dev_actual);
        if (!arena_sp->dev) return fail(RV_ERR_CUDA, "device allocation of the Arrow buffer arena failed");
        res->arenas.assign(res->chunks.size(), arena_sp);
        RV_CUDA(cudaMemsetAsync(arena_sp->dev, 0, std::max<size_t>(L.total_bytes, 64), stream));
        RV_CUDA(cudaStreamSynchronize(stream));
        res->arrow_bytes = exported_bytes(plan, res->chunks);
        *out = res.release();
        return RV_OK;
    }

    DevicePlan dp;
    rv_status st = device_plan(s, device, &dp);
    if (st) return st;
    SchemaStats stats;
    {
        std::lock_guard<std::mutex> g(s->mu);
        stats = s->stats;
    }

    DecodeParams p{};
    p.data = d_data; p.offsets = d_offsets; p.n = n; p.chunk_rows = chunk_rows; p.k = k;
    p.n_streams = S; p.n_slots = n_slots;
    p.sym_off = dp.sym_off; p.sym_bytes = dp.sym_bytes; p.stream_slot = dp.stream_slot;
    p.n_utf8 = 0;
    for (int i = 0; i < S; ++i) p.n_utf8 += plan.streams[size_t(i)].is_rows ? 0 : 1;
    p.frame_skip = uint32_t(std::max(hints.framing.header_bytes, 0));
    p.frame_check = hints.framing.check_magic ? (hints.framing.schema_id >= 0 ? 2 : 1) : 0;
    p.frame_id = uint32_t(hints.framing.schema_id >= 0 ? hints.framing.schema_id : 0);

    // ---- the walker and its tile; shared-memory windows: [fixed tables][input window (+pad)][Utf8 staging / scan area]
    const size_t limit = 227 * 1024;
    int tile = kBlock;          // rows per tile == threads per CTA
    bool use_jit = false;       // schema-specialised walker (NVRTC), else the generic interpreter
    int plan_nodes = 0;         // the generated walker has the plan baked in
    uint32_t item_bytes = 0;
    size_t cur_bytes = 0, fixed = 0;
    int64_t span_hint = -1;     // host path: the largest tile's input span, exactly
    auto set_walker = [&](int tile_, bool jit_) {
        tile = tile_;
        use_jit = jit_;
        plan_nodes = use_jit ? 0 : int(plan.nodes.size());
        cur_bytes = size_t(S) * size_t(tile) * 4;
        // the generated walker's item-position table is one of the fixed tables: it comes out of the two windows' room
        // (configure below gives up the windows' margin where that keeps a CTA per SM)
        item_bytes = use_jit ? item_table_bytes(item_parallel_lists(plan), tile) : 0u;
        fixed = smem_map(plan_nodes, S, n_slots, 0, 0, use_jit, item_bytes, tile).stage;  // everything but the two windows (incl. the pad)
        span_hint = hints.offsets ? max_tile_span(hints.offsets, n, k, tile) : -1;
    };
    auto too_wide = [&] { return fixed + (use_jit ? cur_bytes : 0) + 2048 > limit; };
    // CTAs of `bytes` of shared memory an SM holds; registers allow three 256-row or two 384-row CTAs (80 per thread)
    auto ctas_per_sm = [&](size_t bytes) { const size_t c = (228 * 1024) / (bytes + 1024); return tile > kBlock ? std::min<size_t>(c, 2) : c; };
    size_t smem_bytes = 0;
    auto configure = [&](const SchemaStats& st_) {  // re-evaluated per pass: a measuring pass teaches the next one
        const double in_per_row = hints.total_bytes >= 0 ? double(hints.total_bytes) / double(n) : (st_.in_per_row > 0 ? st_.in_per_row : 128.0);
        unsigned long long max_span = span_hint >= 0 ? static_cast<unsigned long long>(span_hint)
                                      : (st_.max_span ? st_.max_span + st_.max_span / 16 : static_cast<unsigned long long>(in_per_row * tile * 1.25));
        // The window is sized for the LARGEST tile, so that no tile takes the slow global-memory walk; outliers beyond
        // 1.5x the mean tile are not allowed to shrink everyone's occupancy and do take it.
        size_t want_in = std::min<size_t>(size_t(max_span), size_t(in_per_row * tile * env_double("RV_IN_CLAMP", 1.5))) + 48;
        want_in = std::max<size_t>(align_up(want_in, 64), 2048);
        const size_t room = (limit - fixed - 64) & ~size_t(15);
        const size_t min_stage = use_jit ? align_up(cur_bytes, 16) : 0;
        size_t cap_in = std::min(want_in, room - std::min(room, min_stage));
        size_t cap_stage = 0;
        if (p.n_utf8 > 0) {
            // a tile's share of the Utf8 bytes: the largest seen (+6%), else everything the window could hold
            const size_t seen = st_.max_utf8 ? size_t(st_.max_utf8 + st_.max_utf8 / 16) : cap_in + size_t(p.n_utf8) * 31;
            double utf8_per_row = 0;
            if (st_.valid) for (int i = 0; i < S; ++i) if (!plan.streams[size_t(i)].is_rows) utf8_per_row += st_.per_row[size_t(i)];
            size_t want_out = seen;
            if (st_.valid) want_out = std::min<size_t>(seen, size_t(utf8_per_row * tile * env_double("RV_OUT_CLAMP", 1.5)) + size_t(p.n_utf8) * 31);
            cap_stage = align_up(want_out + 64, 64);
            if (const char* ev_ = std::getenv("RV_NO_STAGE_OUT")) if (ev_[0] == '1') cap_stage = 0;
        }
        cap_stage = std::max(cap_stage, min_stage);
        if (cap_in + cap_stage > room) cap_stage = std::max<size_t>(min_stage, (room - cap_in) & ~size_t(15));
        // The windows carry a margin over the largest tile seen (1/16 each).  Where that margin is all that keeps the SM
        // from holding one more CTA — Kafka: windows + the item-position table just above a third of the SM — it is
        // given up, 64 bytes at a time, down to the largest tile seen; otherwise the windows stay as they are.
        if (span_hint < 0 && (st_.max_span || st_.max_utf8)) {
            auto ctas = [&](size_t in_b, size_t st_b) { return ctas_per_sm(smem_map(plan_nodes, S, n_slots, uint32_t(in_b), uint32_t(st_b), use_jit, item_bytes, tile).total); };
            const size_t floor_in = st_.max_span ? std::min(cap_in, std::max<size_t>(align_up(size_t(st_.max_span) + 48, 64), 2048)) : cap_in;
            const size_t floor_stage = st_.max_utf8 ? std::min(cap_stage, std::max(min_stage, size_t(align_up(size_t(st_.max_utf8) + 64, 64)))) : cap_stage;
            const size_t want = ctas(cap_in, cap_stage) + 1;
            size_t in_b = cap_in, st_b = cap_stage;
            while (ctas(in_b, st_b) < want && (in_b > floor_in || st_b > floor_stage)) {
                if (in_b - floor_in >= st_b - floor_stage) in_b = std::max(floor_in, in_b - 64);
                else st_b = std::max(floor_stage, st_b - 64);
            }
            if (ctas(in_b, st_b) >= want) { cap_in = in_b; cap_stage = st_b; }
        }
        p.smem_data_cap = uint32_t(cap_in);
        p.smem_stage_cap = uint32_t(cap_stage);
        const size_t pad_smem = size_t(env_double("RV_SMEM_PAD", 0));  // development knob: occupancy sensitivity
        smem_bytes = std::min<size_t>(smem_map(plan_nodes, S, n_slots, p.smem_data_cap, p.smem_stage_cap, use_jit, item_bytes, tile).total + pad_smem, limit);
        p.prefetch_dist = 0;
        if (!(std::getenv("RV_NO_PREFETCH") && std::getenv("RV_NO_PREFETCH")[0] == '1')) {
            // CTAs resident on the device ~ how far ahead the tile a finishing CTA's successor will take is
            const int ctas = int(std::max<size_t>(1, std::min<size_t>(8, ctas_per_sm(smem_bytes))));
            int sms = 132;
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
            p.prefetch_dist = sms * ctas;
        }
    };
    // The tile.  384 rows (kWideTile) when the walker is the generated one, the plan has more than eight streams and two
    // 384-row CTAs fit an SM: every stream's scan and look-back then has a warp of its own (at 256 rows, eight warps
    // take twelve streams' chains two after one another on four of them), and a third fewer tiles share the per-tile
    // work (prologue, window staging, look-back, write-out) at the same 24 warps per SM.  Otherwise 256 rows.  Two CTAs
    // fit when the windows as configure() sizes them for this call, the 384-row item table and scan area leave 2 x
    // (smem + 1 KiB) within the SM's 228 KiB; __launch_bounds__(384, 2) holds the walker to 80 registers.  A call
    // without history measures first, and its measuring pass stages no strings: it needs the input window and the
    // scan area only.  RV_TILE=256 (development knob) keeps every plan at 256 rows for A/B runs.
    auto choose_tile = [&]() -> JitState {
        const char* ev_ = std::getenv("RV_TILE");
        if (S > kWideStreams && jit_enabled() && !(ev_ && std::atoi(ev_) == kBlock)) {
            set_walker(kWideTile, true);
            if (!too_wide()) {
                const SchemaStats st_ = stats_at(stats, kWideTile, plan);
                configure(st_);
                const size_t need = st_.valid ? smem_bytes
                                              : smem_map(0, S, n_slots, p.smem_data_cap, uint32_t(align_up(cur_bytes, 16)), true, item_bytes, tile).total;
                if (ctas_per_sm(need) >= 2) {
                    const JitState j = ensure_jit(s, device, kWideTile);
                    if (j.ok) return j;
                }
            }
        }
        const JitState j = ensure_jit(s, device, kBlock);
        set_walker(kBlock, j.ok);
        return j;
    };
    const JitState jit = choose_tile();
    t_walker = use_jit ? "jit" : "interp";
    t_tile = tile;
    if (too_wide()) return fail(RV_ERR_SCHEMA, "schema too wide for the shared-memory cursor table");

    const int64_t tpc = std::max<int64_t>(1, (chunk_rows + tile - 1) / tile);
    const int64_t tiles_last = (last_rows + tile - 1) / tile;
    const int64_t n_tiles = tpc * (k - 1) + tiles_last;
    if (n_tiles > 0x7FFFFFF0ll) return fail(RV_ERR_INVALID, "too many records for one call");
    p.tiles_per_chunk = int32_t(tpc); p.n_tiles = int32_t(n_tiles);
    p.nodes = dp.nodes; p.n_nodes = int32_t(plan_nodes);

    // ---- per-call device state: [ctrl][bufs table][caps][null-count jobs][ones] in ONE block, initialised by one
    // copy from a pinned template and (ctrl + ones) read back by one copy ------------------------------------
    const int nv = int(plan.validity_slots.size());
    const size_t ctrl_words = size_t(CW_CHUNK_TOT) + chunk_tot.size();
    const size_t off_ctrl = 0;
    const size_t off_ones = align_up(off_ctrl + ctrl_words * 8, 16);
    const size_t ones_n = size_t(k) * size_t(std::max(nv, 1));
    const size_t back_bytes = off_ones + ones_n * 8;               // the part that is read back
    const size_t off_bufs = align_up(back_bytes, 16);
    const size_t off_caps = align_up(off_bufs + size_t(k) * size_t(n_slots) * sizeof(void*), 16);
    const size_t off_jobs = align_up(off_caps + size_t(k) * size_t(Sx) * 4, 16);
    const size_t misc_bytes = align_up(off_jobs + size_t(k) * size_t(std::max(nv, 1)) * sizeof(NullCountJob), 16);
    uint8_t* h_misc = t_scratch.get(misc_bytes + back_bytes);
    if (!h_misc) return fail(RV_ERR_CUDA, "pinned allocation of the call state failed");
    uint8_t* h_back = h_misc + misc_bytes;
    DevBuf d_misc, d_state;
    RV_CUDA(d_misc.alloc(misc_bytes, stream));
    RV_CUDA(d_state.alloc(size_t(Sx) * size_t(n_tiles) * 8, stream));
    SyncOnExit guard{stream};  // declared after the cached device blocks: runs before they go back to the cache
    uint8_t* dm = static_cast<uint8_t*>(d_misc.p);
    p.ctrl = reinterpret_cast<unsigned long long*>(dm + off_ctrl);
    p.tile_state = static_cast<unsigned long long*>(d_state.p);
    cudaEvent_t* ev = nullptr;
    RV_CUDA(t_events.get(device, &ev));
    mark("setup");

    // chunk j's rows
    auto rows_of = [&](int j) { return j == k - 1 ? last_rows : chunk_rows; };
    std::vector<unsigned long long> caps(chunk_tot.size(), 0ull);
    bool exact_caps = false;
    bool count_only = !stats.valid;
    if (stats.valid) {
        const double margin = env_double("RV_CAP_MARGIN", 1.10);
        // What the input can possibly hold bounds the plan (history from a batch of a few huge records must not size the
        // buffers of a batch of millions): every string byte and every list item costs at least one input byte.
        const double in_bytes = hints.total_bytes >= 0 ? double(hints.total_bytes) : double(n) * stats.in_per_row * 2.0 + 65536.0;
        double planned = 0;
        for (int j = 0; j < k; ++j)
            for (int i = 0; i < S; ++i) {
                double want = double(rows_of(j)) * stats.per_row[size_t(i)] * margin + 4096.0;
                const Stream& st_ = plan.streams[size_t(i)];
                const bool enum_text = !st_.is_rows && (plan.nodes[size_t(st_.node)].kind == NK_ENUM ||
                                                        plan.nodes[size_t(st_.node)].kind == NK_DEFAULT);  // symbol / default text is not input bytes
                if (!enum_text) want = std::min(want, in_bytes + 4096.0);
                caps[size_t(j) * size_t(Sx) + size_t(i)] = static_cast<unsigned long long>(std::min(want, 2147483647.0));
                planned += want;
            }
        // a plan far beyond anything the input could produce (stale history): measure first instead
        if (planned > 64.0 * in_bytes + double(size_t(1) << 30)) count_only = true;
    }
    Layout capL;
    std::vector<long long> ones(ones_n, 0);
    unsigned long long* hb_ctrl = reinterpret_cast<unsigned long long*>(h_back + off_ctrl);

    for (int pass = 0; pass < 3; ++pass) {
        ++t_passes;
        configure(stats_at(stats, tile, plan));
        if (trace)
            trace_line += "tile=" + std::to_string(tile) + " smem=" + std::to_string(smem_bytes) + "(in " + std::to_string(p.smem_data_cap) + " stage " + std::to_string(p.smem_stage_cap) +
                          " items " + std::to_string(item_bytes) + "; largest tile seen: span " + std::to_string(stats.max_span) +
                          " utf8 " + std::to_string(stats.max_utf8) + ") ";
        // ---- arena for this pass's capacities
        uint8_t* arena = nullptr;
        if (!count_only) {
            capL = compute_layout(plan, n, k, caps.data());
            arena_sp->drop_device();
            arena_sp->bytes = capL.total_bytes;
            arena_sp->dev = devmem().get(std::max<size_t>(capL.total_bytes, 64), device, &arena_sp->dev_actual);
            if (!arena_sp->dev) {
                // the planned arena does not fit: measure, then allocate exactly what the data needs
                if (!exact_caps) { count_only = true; }
                else return fail(RV_ERR_CUDA, "device allocation of the Arrow buffer arena failed (" + std::to_string(capL.total_bytes) + " bytes)");
            } else {
                arena = static_cast<uint8_t*>(arena_sp->dev);
            }
        }
        // ---- template of the call state
        std::memset(h_misc, 0, misc_bytes);
        unsigned long long* hc = reinterpret_cast<unsigned long long*>(h_misc + off_ctrl);
        hc[CW_ERR] = ~0ull;
        hc[CW_MAX_SPAN] = stats.tile == tile ? stats.max_span : 0ull;   // the kernel only raises these
        hc[CW_MAX_UTF8] = stats.tile == tile ? stats.max_utf8 : 0ull;
        if (!count_only) {
            void** hb = reinterpret_cast<void**>(h_misc + off_bufs);
            for (int j = 0; j < k; ++j)
                for (int sl = 0; sl < n_slots; ++sl) hb[size_t(j) * size_t(n_slots) + size_t(sl)] = arena + capL.chunks[size_t(j)].slot_off[size_t(sl)];
            uint32_t* hcap = reinterpret_cast<uint32_t*>(h_misc + off_caps);
            for (size_t i = 0; i < caps.size(); ++i) hcap[i] = uint32_t(caps[i]);
            NullCountJob* jobs = reinterpret_cast<NullCountJob*>(h_misc + off_jobs);
            for (int j = 0; j < k; ++j)
                for (int v = 0; v < nv; ++v) {
                    const int sl = plan.validity_slots[size_t(v)];
                    const int space = plan.slots[size_t(sl)].space;
                    NullCountJob& job = jobs[size_t(j) * size_t(nv) + size_t(v)];
                    job.bitmap = reinterpret_cast<const uint32_t*>(arena + capL.chunks[size_t(j)].slot_off[size_t(sl)]);
                    job.n_bits = rows_of(j);
                    job.n_bits_dev = space == 0 ? nullptr : p.ctrl + CW_CHUNK_TOT + size_t(j) * size_t(Sx) + size_t(plan.space_stream[size_t(space)]);
                }
        }
        p.bufs = count_only ? nullptr : reinterpret_cast<void* const*>(dm + off_bufs);
        p.caps = count_only ? nullptr : reinterpret_cast<const uint32_t*>(dm + off_caps);
        p.count_only = count_only ? 1 : 0;

        RV_CUDA(cudaMemcpyAsync(dm, h_misc, misc_bytes, cudaMemcpyHostToDevice, stream));
        RV_CUDA(cudaMemsetAsync(d_state.p, 0, size_t(Sx) * size_t(n_tiles) * 8, stream));
        if (!count_only && capL.zero_bytes) RV_CUDA(cudaMemsetAsync(arena, 0, capL.zero_bytes, stream));
        RV_CUDA(cudaEventRecord(ev[0], stream));
        if (use_jit) {
            void* args[] = {&p};
            const cudaError_t le = cudaLaunchKernel(reinterpret_cast<const void*>(jit.fused), dim3(unsigned(p.n_tiles)), dim3(unsigned(tile)), args, smem_bytes, stream);
            if (le != cudaSuccess) {
                // the driver rejected the specialised kernel (attributes, architecture): remember it for this
                // (schema, device) and decode this call with the interpreter kernel instead — still on the GPU
                (void)cudaGetLastError();
                {
                    std::lock_guard<std::mutex> g(s->mu);
                    JitState& j = s->jit[{device, tile}];
                    j.ok = false;
                    j.status = std::string("launch of the compiled walker was rejected: ") + cudaGetErrorString(le);
                }
                RV_CUDA(cudaStreamSynchronize(stream));
                return decode_on_device(s, d_data, d_offsets, n, num_chunks, hints, stream, device, out, record_base);
            }
        } else {
            launch_fused(p, smem_bytes, stream);
        }
        RV_CUDA(cudaEventRecord(ev[1], stream));
        t_launches += 1;
        if (!count_only && nv > 0) {
            launch_null_count(reinterpret_cast<const NullCountJob*>(dm + off_jobs), k * nv, reinterpret_cast<long long*>(dm + off_ones), stream);
            t_launches += 1;
        }
        RV_CUDA(cudaEventRecord(ev[2], stream));
        RV_CUDA(cudaGetLastError());
        RV_CUDA(cudaMemcpyAsync(h_back, dm, back_bytes, cudaMemcpyDeviceToHost, stream));
        mark("launched");
        RV_CUDA(cudaStreamSynchronize(stream));
        mark("sync");

        const unsigned long long err_word = hb_ctrl[CW_ERR];
        if (err_word != ~0ull) {
            const uint32_t code = uint32_t(err_word & 0xFF);
            return fail(status_of(code), std::string(err_text(code)) + " (record " + std::to_string(int64_t(err_word >> 8) + record_base) + ")");
        }
        std::memcpy(chunk_tot.data(), hb_ctrl + CW_CHUNK_TOT, chunk_tot.size() * 8);
        const bool over = hb_ctrl[CW_OVER] != 0ull;
        t_slow_tiles = (long long)hb_ctrl[CW_SLOW_TILES];
        float ms = 0;
        cudaEventElapsedTime(&ms, ev[0], ev[1]);
        // ---- remember what this call needed
        {
            std::lock_guard<std::mutex> g(s->mu);
            SchemaStats& ss = s->stats;
            if (ss.per_row.size() != size_t(S)) ss.per_row.assign(size_t(S), 0.0);
            for (int i = 0; i < S; ++i) {
                double worst = 0;  // the densest chunk decides: every chunk's buffers must hold
                for (int j = 0; j < k; ++j) worst = std::max(worst, double(chunk_tot[size_t(j) * size_t(Sx) + size_t(i)]) / double(std::max<int64_t>(rows_of(j), 1)));
                double& r = ss.per_row[size_t(i)];
                r = (!ss.valid || worst > r) ? worst : r * 0.9 + worst * 0.1;
            }
            if (hints.total_bytes >= 0) ss.in_per_row = double(hints.total_bytes) / double(n);
            else if (hb_ctrl[CW_IN_LAST] >= hb_ctrl[CW_IN_FIRST]) ss.in_per_row = double(hb_ctrl[CW_IN_LAST] - hb_ctrl[CW_IN_FIRST]) / double(n);
            if (ss.tile != tile) ss.max_span = ss.max_utf8 = 0;  // largest tiles are per tile size: measured afresh
            ss.max_span = std::max(ss.max_span, hb_ctrl[CW_MAX_SPAN]);
            ss.max_utf8 = std::max(ss.max_utf8, hb_ctrl[CW_MAX_UTF8]);
            ss.tile = tile;
            ss.valid = true;
            stats = ss;
        }
        if (!count_only && !over) {
            t_timings[0] = ms;
            cudaEventElapsedTime(&t_timings[3], ev[1], ev[2]);
            std::memcpy(ones.data(), h_back + off_ones, ones_n * 8);
            break;
        }
        // the pass only measured (first call on the schema, or the data outgrew the plan): repeat with exact sizes
        t_timings[1] += ms;
        if (exact_caps) return fail(RV_ERR_CUDA, "internal error: exact-size pass reported a capacity overflow");
        caps = chunk_tot;
        exact_caps = true;
        count_only = false;
    }

    // ---- exact logical sizes on top of the capacity-planned placement ---------------------------
    Layout L = compute_layout(plan, n, k, chunk_tot.data());
    for (int j = 0; j < k; ++j) L.chunks[size_t(j)].slot_off = capL.chunks[size_t(j)].slot_off;
    res->chunks = std::move(L.chunks);
    res->arenas.assign(res->chunks.size(), arena_sp);
    for (int j = 0; j < k; ++j)
        for (int v = 0; v < nv; ++v) {
            const int sl = plan.validity_slots[size_t(v)];
            ChunkOut& c = res->chunks[size_t(j)];
            c.null_count[size_t(sl)] = c.space_rows[size_t(plan.slots[size_t(sl)].space)] - ones[size_t(j) * size_t(nv) + size_t(v)];
        }
    res->arrow_bytes = exported_bytes(plan, res->chunks);
    mark("finish");
    if (trace) std::fprintf(stderr, "[rv trace] passes=%d %s\n", t_passes, trace_line.c_str());
    guard.armed = false;  // the last pass synchronised the stream
    *out = res.release();
    return RV_OK;
}

rv_status check_decodable(const rv_schema* s) {
    if (!s) return fail(RV_ERR_INVALID, "null schema handle");
    if (!s->supported)
        return fail(RV_ERR_SCHEMA, "schema is outside the direct-decode subset (" + s->why + "); this library has no Value-tree CPU fallback");
    if (!s->has_plan) return fail(RV_ERR_SCHEMA, s->why);
    return RV_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
extern "C" {

rv_status rv_schema_parse(const char* json, size_t len, rv_schema** out) {
    if (!json || !out) return fail(RV_ERR_INVALID, "null argument");
    *out = nullptr;
    try {
        auto s = std::make_unique<rv_schema>();
        s->avro = parse_avro_schema(json, len);
        s->supported = is_supported(*s->avro, &s->why);
        if (s->avro->k == AK::Record) {
            try {
                s->fields = to_arrow_fields(*s->avro);
                s->has_fields = true;
            } catch (const std::exception& e) {
                if (s->supported) { s->supported = false; s->why = e.what(); }
            }
        }
        if (s->supported && s->has_fields) {
            try {
                s->plan = build_plan(*s->avro, s->fields);
                s->has_plan = true;
            } catch (const std::exception& e) {
                s->why = e.what();
            }
        }
        *out = s.release();
        return RV_OK;
    } catch (const std::exception& e) {
        return fail(RV_ERR_SCHEMA, e.what());
    }
}

rv_schema* rv_schema_retain(rv_schema* s) {
    if (s) s->refs.fetch_add(1, std::memory_order_relaxed);
    return s;
}

void rv_schema_release(rv_schema* s) {
    if (!s) return;
    if (s->refs.fetch_sub(1, std::memory_order_acq_rel) == 1) {
        for (auto& kv : s->dev) {
            cudaFree(kv.second.nodes);
            cudaFree(kv.second.sym_off);
            cudaFree(kv.second.sym_bytes);
            cudaFree(kv.second.stream_slot);
        }
        for (auto& kv : s->jit)
            if (kv.second.lib) cudaLibraryUnload(kv.second.lib);
        (void)cudaGetLastError();
        delete s;
    }
}

int rv_schema_is_supported(const rv_schema* s) { return s && s->supported && s->has_plan ? 1 : 0; }

rv_status rv_schema_project(const rv_schema* s, const char* const* columns, int64_t n_columns, rv_schema** out) {
    if (!s || !out || (!columns && n_columns != 0) || n_columns < 0) return fail(RV_ERR_INVALID, "null argument");
    *out = nullptr;
    rv_status st = check_decodable(s);
    if (st) return st;
    std::vector<std::string> names, requested;
    for (const ArrowField& f : s->fields) names.push_back(f.name);
    for (int64_t i = 0; i < n_columns; ++i) {
        if (!columns[i]) return fail(RV_ERR_INVALID, "column projection: null column name");
        requested.emplace_back(columns[i]);
    }
    try {
        const std::vector<int> sel = select_columns(names, requested);
        auto p = std::make_unique<rv_schema>();
        p->avro = s->avro;
        p->supported = true;
        p->has_fields = true;
        p->reader = s->reader;
        p->res = s->res;
        const AvroNode& out_schema = s->res ? *s->reader : *s->avro;  // (a resolved handle's columns are the reader's fields)
        std::vector<ArrowField> all = s->keep.empty() ? s->fields : to_arrow_fields(out_schema);
        for (int i : sel) {
            p->keep.push_back(s->keep.empty() ? i : s->keep[size_t(i)]);  // (a projection of a projection: fields of the schema)
            p->fields.push_back(s->fields[size_t(i)]);
        }
        p->plan = p->res ? build_resolved_plan(*p->res, all, &p->keep) : build_plan(*p->avro, all, &p->keep);
        p->has_plan = true;
        *out = p.release();
        return RV_OK;
    } catch (const std::invalid_argument& e) {
        return fail(RV_ERR_INVALID, e.what());
    } catch (const std::exception& e) {
        return fail(RV_ERR_SCHEMA, e.what());
    }
}

rv_status rv_schema_resolve(const rv_schema* writer, const rv_schema* reader, rv_schema** out) {
    if (!writer || !reader || !out) return fail(RV_ERR_INVALID, "null argument");
    *out = nullptr;
    if (!writer->keep.empty() || writer->res || !reader->keep.empty() || reader->res)
        return fail(RV_ERR_INVALID, "schema resolution: pass the handles of the writer's and the reader's full schemas (rv_schema_parse)");
    rv_status st = check_decodable(writer);
    if (st) return st;
    st = check_decodable(reader);
    if (st) return st;
    try {
        auto p = std::make_unique<rv_schema>();
        p->avro = writer->avro;
        p->reader = reader->avro;
        p->res = std::make_shared<const Resolution>(resolve_schemas(*p->avro, *p->reader));
        p->supported = true;
        p->fields = reader->fields;
        p->has_fields = true;
        p->plan = build_resolved_plan(*p->res, p->fields);
        p->has_plan = true;
        *out = p.release();
        return RV_OK;
    } catch (const std::exception& e) {
        return fail(RV_ERR_SCHEMA, e.what());
    }
}

rv_status rv_schema_export_arrow(const rv_schema* s, struct ArrowSchema* out) {
    if (!s || !out) return fail(RV_ERR_INVALID, "null argument");
    if (!s->has_fields) return fail(RV_ERR_SCHEMA, s->why.empty() ? "top-level schema is not a record" : s->why);
    try {
        export_arrow_schema(s->fields, out);
        return RV_OK;
    } catch (const std::exception& e) {
        return fail(RV_ERR_SCHEMA, e.what());
    }
}

static rv_status framing_ok(const rv_framing* f) {
    if (!f) return RV_OK;
    if (f->header_bytes < 0 || f->header_bytes > 4096) return fail(RV_ERR_INVALID, "framing: header_bytes out of range");
    if (f->check_magic && f->header_bytes < 5) return fail(RV_ERR_INVALID, "framing: the Confluent header check needs header_bytes >= 5");
    if (f->schema_id > int64_t(0xFFFFFFFFu)) return fail(RV_ERR_INVALID, "framing: schema_id is a u32");
    return RV_OK;
}

rv_status rv_decode_device_framed(const rv_schema* s, const uint8_t* d_data, const int64_t* d_offsets, int64_t n,
                                  int64_t num_chunks, const rv_framing* framing, void* cuda_stream, rv_result** out) {
    if (!out) return fail(RV_ERR_INVALID, "null argument");
    *out = nullptr;
    rv_status st = check_decodable(s);
    if (st) return st;
    st = framing_ok(framing);
    if (st) return st;
    if (n < 0 || (n > 0 && (!d_data || !d_offsets))) return fail(RV_ERR_INVALID, "bad input pointers");
    if (reinterpret_cast<uintptr_t>(d_data) & 15u) return fail(RV_ERR_INVALID, "d_data must be 16-byte aligned");
    int device = 0;
    st = ensure_cuda(&device);
    if (st) return st;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    InputHints hints;
    if (framing) hints.framing = *framing;
    try {
        st = decode_on_device(const_cast<rv_schema*>(s), d_data, d_offsets, n, num_chunks, hints, stream, device, out);
    } catch (const std::exception& e) {
        st = fail(RV_ERR_INVALID, e.what());
    }
    // error paths hand cached device blocks back: nothing may still be running on them
    if (st) { const std::string keep = t_error; cudaStreamSynchronize(stream); (void)cudaGetLastError(); t_error = keep; }
    return st;
}

rv_status rv_decode_device(const rv_schema* s, const uint8_t* d_data, const int64_t* d_offsets, int64_t n,
                           int64_t num_chunks, void* cuda_stream, rv_result** out) {
    return rv_decode_device_framed(s, d_data, d_offsets, n, num_chunks, nullptr, cuda_stream, out);
}

}  // extern "C"

namespace {

// Brings one arena to a pinned host slab on `stream`: the capacity-planned device arena is packed into an
// exact-size one (device -> device, compact_kernel), that one is copied down, and BOTH device blocks go back to the
// cache — a host batch keeps only its pinned slab alive.  Rewrites the chunks' slot offsets to the exact layout.
rv_status arena_to_host(rv_result& r, Arena& a, cudaStream_t stream, float* ms) {
    if (a.host) return RV_OK;
    const Plan& plan = r.schema->plan;
    const int n_slots = int(plan.slots.size());
    // exact layout over the chunks this arena backs
    std::vector<size_t> mine;
    for (size_t i = 0; i < r.chunks.size(); ++i)
        if (r.arenas[i].get() == &a) mine.push_back(i);
    size_t total = 0;
    std::vector<CompactJob> jobs;
    std::vector<std::vector<size_t>> new_off(mine.size(), std::vector<size_t>(size_t(n_slots), 0));
    const uint8_t* src = static_cast<const uint8_t*>(a.dev);
    for (int pass = 0; pass < 2; ++pass)  // same order as compute_layout: zero-initialised bit buffers first
        for (size_t mi = 0; mi < mine.size(); ++mi) {
            const ChunkOut& c = r.chunks[mine[mi]];
            for (int sl = 0; sl < n_slots; ++sl) {
                const Slot& slot = plan.slots[size_t(sl)];
                if (slot.zero_init != (pass == 0)) continue;
                size_t bytes = size_t(c.slot_bytes[size_t(sl)]);
                if (slot.role == SlotRole::Validity || slot.role == SlotRole::Bits) bytes = size_t((c.space_rows[size_t(slot.space)] + 31) / 32) * 4;
                new_off[mi][size_t(sl)] = total;
                if (bytes) jobs.push_back(CompactJob{src + c.slot_off[size_t(sl)], reinterpret_cast<uint8_t*>(total), int64_t(bytes)});  // dst: offset for now
                total += (std::max<size_t>(bytes, 1) + 63) & ~size_t(63);
            }
        }
    const size_t host_bytes = std::max<size_t>(total, 64);
    size_t actual = 0;
    void* h = pinned().get(host_bytes, &actual);
    if (!h) return fail(RV_ERR_CUDA, "pinned host allocation failed");
    DevBuf packed, d_jobs;
    cudaError_t e = packed.alloc(host_bytes, stream);
    if (e == cudaSuccess) e = d_jobs.alloc(std::max<size_t>(jobs.size(), 1) * sizeof(CompactJob), stream);
    uint8_t* h_jobs = t_scratch.get(std::max<size_t>(jobs.size(), 1) * sizeof(CompactJob));
    if (e != cudaSuccess || !h_jobs) { pinned().put(h, actual); return fail(RV_ERR_CUDA, "device allocation for the host export failed"); }
    SyncOnExit guard{stream};
    for (CompactJob& job : jobs) job.dst = static_cast<uint8_t*>(packed.p) + reinterpret_cast<size_t>(job.dst);
    std::memcpy(h_jobs, jobs.data(), jobs.size() * sizeof(CompactJob));
    cudaEvent_t* ev = nullptr;
    e = t_events.get(a.device, &ev);
    if (e == cudaSuccess && !jobs.empty()) e = cudaMemcpyAsync(d_jobs.p, h_jobs, jobs.size() * sizeof(CompactJob), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess && !jobs.empty()) {
        const int parts = int(std::max<size_t>(1, std::min<size_t>(64, (total / std::max<size_t>(jobs.size(), 1)) >> 16)));
        launch_compact(static_cast<const CompactJob*>(d_jobs.p), int(jobs.size()), parts, stream);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaEventRecord(ev[6], stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h, packed.p, host_bytes, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaEventRecord(ev[7], stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) {
        (void)cudaStreamSynchronize(stream);
        (void)cudaGetLastError();
        pinned().put(h, actual);
        return fail(RV_ERR_CUDA, std::string("device->host copy: ") + cudaGetErrorString(e));
    }
    float t = 0;
    cudaEventElapsedTime(&t, ev[6], ev[7]);
    if (ms) *ms += t;
    guard.armed = false;
    a.host = h;
    a.host_actual = actual;
    a.host_bytes = host_bytes;
    a.drop_device();
    for (size_t mi = 0; mi < mine.size(); ++mi) r.chunks[mine[mi]].slot_off = new_off[mi];
    return RV_OK;
}

// H2D of rows [r0, r1) of the caller's packed input, decode into `num_chunks` batches, D2H.
rv_status decode_host_range(rv_schema* s, const uint8_t* data, const int64_t* offsets, int64_t r0, int64_t r1, int64_t num_chunks,
                            cudaStream_t stream, int device, rv_result** out, float* h2d_ms, float* d2h_ms, const rv_framing& framing) {
    const int64_t n = r1 - r0;
    DevBuf d_data, d_off;
    InputHints hints;
    hints.framing = framing;
    const uint8_t* base = nullptr;
    rv_status st = RV_OK;
    if (n > 0) {
        const int64_t b0 = offsets[r0];
        const int64_t total = offsets[r1] - b0;
        if (total < 0) return fail(RV_ERR_INVALID, "offsets are not monotonic");
        hints.total_bytes = total;
        hints.offsets = offsets + r0;  // the largest tile span, exactly (the host can read the offsets): sizes the window
        RV_CUDA(d_data.alloc(size_t(total) + 64, stream));
        RV_CUDA(d_off.alloc(size_t(n + 1) * 8, stream));
        cudaEvent_t* ev = nullptr;
        RV_CUDA(t_events.get(device, &ev));
        cudaEventRecord(ev[4], stream);
        // The device copy keeps the caller's absolute offsets: the base pointer is biased so that
        // base + offsets[i] addresses record i (kept 16-byte aligned by the b0 & 15 shift).
        cudaError_t e = upload(static_cast<uint8_t*>(d_data.p) + (b0 & 15), data + b0, size_t(total), device, stream);
        if (e == cudaSuccess) e = upload(static_cast<uint8_t*>(d_off.p), reinterpret_cast<const uint8_t*>(offsets + r0), size_t(n + 1) * 8, device, stream);
        cudaEventRecord(ev[5], stream);
        if (e != cudaSuccess) { (void)cudaStreamSynchronize(stream); return fail(RV_ERR_CUDA, std::string("host->device copy: ") + cudaGetErrorString(e)); }
        base = static_cast<const uint8_t*>(d_data.p) + (b0 & 15) - b0;
    }
    try {
        st = decode_on_device(s, base, static_cast<const int64_t*>(d_off.p), n, num_chunks, hints, stream, device, out, r0);
    } catch (const std::exception& e) {
        st = fail(RV_ERR_INVALID, e.what());
    }
    if (st) { const std::string keep = t_error; cudaStreamSynchronize(stream); (void)cudaGetLastError(); t_error = keep; return st; }
    if (n > 0 && h2d_ms) {
        cudaEvent_t* ev = nullptr;
        float t = 0;
        if (t_events.get(device, &ev) == cudaSuccess && cudaEventElapsedTime(&t, ev[4], ev[5]) == cudaSuccess) *h2d_ms += t;
        (void)cudaGetLastError();
    }
    st = arena_to_host(**out, *(*out)->arenas[0], stream, d2h_ms);
    if (st) { rv_result_free(*out); *out = nullptr; }
    return st;
}

bool pipeline_enabled() {
    const char* e = std::getenv("RV_PIPELINE");
    return !(e && e[0] == '0');
}

// ---- persistent chunk workers ---------------------------------------------------------------------
// The host path decodes the chunks of a call (independent batches) on a few long-lived threads per device, each
// with its own stream, events and pinned scratch, so that the H2D copy of chunk i+1 overlaps the kernels and the
// D2H copy of chunk i.  (Spawning threads per call re-created all of that every time.)
class WorkerPool {
  public:
    explicit WorkerPool(int device, int n) : device_(device) {
        for (int w = 0; w < n; ++w) std::thread([this, w] { run(w); }).detach();
    }
    void submit(std::function<void(cudaStream_t)> fn) {
        { std::lock_guard<std::mutex> g(mu_); q_.push_back(std::move(fn)); }
        cv_.notify_one();
    }

  private:
    void run(int w) {
        cudaSetDevice(device_);
        bind_thread_to_gpu_node(device_);
        cudaStream_t stream = worker_stream(device_, w);
        for (;;) {
            std::function<void(cudaStream_t)> fn;
            {
                std::unique_lock<std::mutex> g(mu_);
                cv_.wait(g, [&] { return !q_.empty(); });
                fn = std::move(q_.front());
                q_.pop_front();
            }
            fn(stream);
        }
    }
    int device_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<std::function<void(cudaStream_t)>> q_;
};

int worker_count() {
    int want = 4;
    if (const char* ev = std::getenv("RV_WORKERS")) want = std::max(1, std::atoi(ev));
    return std::min(want, 16);
}

WorkerPool& worker_pool(int device) {
    static std::mutex mu;
    static std::map<int, WorkerPool*> pools;  // intentionally leaked: the threads live until the process ends
    std::lock_guard<std::mutex> g(mu);
    auto it = pools.find(device);
    if (it != pools.end()) return *it->second;
    WorkerPool* p = new WorkerPool(device, worker_count());
    pools[device] = p;
    return *p;
}

}  // namespace


// ---- multi-GPU gather (gather.hpp; pyruhvro_b200/distributed.py drives it) -----------------------------------------
struct rv_gather {
    rv_schema* schema = nullptr;
    GatherPlan plan;
    std::vector<std::shared_ptr<Arena>> arenas;  // per group; set on the group's leader by rv_gather_alloc
    ~rv_gather() { if (schema) rv_schema_release(schema); }
};

extern "C" {

int64_t rv_gather_meta_len(const rv_schema* s) { return s && s->has_plan ? gather_meta_len(s->plan) : -1; }

rv_status rv_result_gather_meta(const rv_result* r, int64_t batch, int64_t* out, int64_t cap) {
    if (!r || !out || batch < 0 || batch >= int64_t(r->chunks.size())) return fail(RV_ERR_INVALID, "bad argument");
    if (cap < gather_meta_len(r->schema->plan)) return fail(RV_ERR_INVALID, "meta buffer too small");
    gather_meta_of(r->schema->plan, r->chunks[size_t(batch)], out);
    return RV_OK;
}

rv_status rv_gather_plan(const rv_schema* s, const int64_t* metas, int world, rv_gather** out) {
    if (!s || !s->has_plan || !metas || world < 1 || !out) return fail(RV_ERR_INVALID, "bad argument");
    try {
        auto g = std::make_unique<rv_gather>();
        g->schema = rv_schema_retain(const_cast<rv_schema*>(s));
        g->plan = plan_gather(s->plan, metas, world);
        g->arenas.resize(g->plan.groups.size());
        *out = g.release();
        return RV_OK;
    } catch (const std::exception& e) {
        return fail(RV_ERR_OVERFLOW, e.what());
    }
}

int rv_gather_num_groups(const rv_gather* g) { return g ? int(g->plan.groups.size()) : 0; }
int rv_gather_group_of_rank(const rv_gather* g, int rank) {
    return g && rank >= 0 && rank < int(g->plan.group_of_rank.size()) ? g->plan.group_of_rank[size_t(rank)] : -1;
}

// out[0] = first (leader) rank, out[1] = ranks in the group, out[2] = arena bytes, out[3] = rows of the gathered batch,
// out[4] = bytes the non-leader members push (what crosses NVLink into the leader)
rv_status rv_gather_group_info(const rv_gather* g, int group, int64_t* out) {
    if (!g || !out || group < 0 || group >= int(g->plan.groups.size())) return fail(RV_ERR_INVALID, "bad argument");
    const GatherGroup& gg = g->plan.groups[size_t(group)];
    out[0] = gg.first_rank; out[1] = gg.n_ranks; out[2] = int64_t(gg.arena_bytes); out[3] = gg.out.rows;
    int64_t remote = 0;
    for (size_t m = 1; m < gg.jobs.size(); ++m)
        for (const GatherJob& j : gg.jobs[m]) remote += j.kind == GK_RAW ? j.count : (j.kind == GK_OFFSETS ? 4 * j.count : (j.count + 7) / 8);
    out[4] = remote;
    return RV_OK;
}

// Leader of `group`: allocates the gathered arena, zeroes it (bitmap seams are OR-merged, offsets[0] = 0) and returns
// its device pointer.  Synchronises `cuda_stream`: the pointer may be handed to the peers right away.
rv_status rv_gather_alloc(rv_gather* g, int group, void* cuda_stream, void** out_ptr) {
    if (!g || !out_ptr || group < 0 || group >= int(g->plan.groups.size())) return fail(RV_ERR_INVALID, "bad argument");
    int device = 0;
    rv_status st = ensure_cuda(&device);
    if (st) return st;
    auto a = std::make_shared<Arena>();
    a->device = device;
    a->bytes = g->plan.groups[size_t(group)].arena_bytes;
    a->dev = devmem().get(std::max<size_t>(a->bytes, 64), device, &a->dev_actual);
    if (!a->dev) return fail(RV_ERR_CUDA, "device allocation of the gathered arena failed (" + std::to_string(a->bytes) + " bytes)");
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    RV_CUDA(cudaMemsetAsync(a->dev, 0, std::max<size_t>(a->bytes, 64), stream));
    RV_CUDA(cudaStreamSynchronize(stream));
    g->arenas[size_t(group)] = a;
    *out_ptr = a->dev;
    return RV_OK;
}

// Member `rank` of `group`: pushes batch `batch` of its device-resident result into the gathered arena at `dst_base`
// (its own memory on the leader, peer memory elsewhere) with ONE kernel; synchronises `cuda_stream`.
rv_status rv_gather_push(rv_gather* g, int group, int rank, rv_result* mine, int64_t batch, void* dst_base, void* cuda_stream) {
    if (!g || !mine || !dst_base || group < 0 || group >= int(g->plan.groups.size())) return fail(RV_ERR_INVALID, "bad argument");
    const GatherGroup& gg = g->plan.groups[size_t(group)];
    const int m = rank - gg.first_rank;
    if (m < 0 || m >= gg.n_ranks || batch < 0 || batch >= int64_t(mine->chunks.size())) return fail(RV_ERR_INVALID, "rank / batch outside the group");
    Arena& a = *mine->arenas[size_t(batch)];
    if (!a.dev) return fail(RV_ERR_INVALID, "the shard's batch must be device-resident");
    const ChunkOut& c = mine->chunks[size_t(batch)];
    const std::vector<GatherJob>& jobs = gg.jobs[size_t(m)];
    if (jobs.empty()) return RV_OK;
    std::vector<PushJob> pj(jobs.size());
    int64_t bytes = 0;
    for (size_t i = 0; i < jobs.size(); ++i) {
        const GatherJob& j = jobs[i];
        pj[i] = PushJob{static_cast<const uint8_t*>(a.dev) + c.slot_off[size_t(j.slot)], static_cast<uint8_t*>(dst_base) + j.dst_off, j.count, j.param, j.kind, 0};
        bytes += j.kind == GK_RAW ? j.count : (j.kind == GK_OFFSETS ? 4 * j.count : j.count / 8);
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    DevBuf d_jobs;
    RV_CUDA(d_jobs.alloc(pj.size() * sizeof(PushJob), stream));
    SyncOnExit guard{stream};
    uint8_t* h = t_scratch.get(pj.size() * sizeof(PushJob));
    if (!h) return fail(RV_ERR_CUDA, "pinned allocation failed");
    std::memcpy(h, pj.data(), pj.size() * sizeof(PushJob));
    RV_CUDA(cudaMemcpyAsync(d_jobs.p, h, pj.size() * sizeof(PushJob), cudaMemcpyHostToDevice, stream));
    const int parts = int(std::max<int64_t>(1, std::min<int64_t>(128, (bytes / int64_t(pj.size())) >> 16)));
    launch_gather_push(static_cast<const PushJob*>(d_jobs.p), int(pj.size()), parts, stream);
    RV_CUDA(cudaGetLastError());
    RV_CUDA(cudaStreamSynchronize(stream));
    guard.armed = false;
    t_launches = 1;
    return RV_OK;
}

// Leader of `group`, after every member pushed (the caller's barrier): the gathered batch as a device-resident result
// (rv_result_to_host / rv_result_export / rv_result_export_device apply).
rv_status rv_gather_finish(rv_gather* g, int group, rv_result** out) {
    if (!g || !out || group < 0 || group >= int(g->plan.groups.size())) return fail(RV_ERR_INVALID, "bad argument");
    if (!g->arenas[size_t(group)]) return fail(RV_ERR_INVALID, "rv_gather_alloc was not called for this group on this rank");
    auto res = std::make_unique<rv_result>();
    res->schema = rv_schema_retain(g->schema);
    res->chunks.push_back(g->plan.groups[size_t(group)].out);
    res->arenas.push_back(g->arenas[size_t(group)]);
    res->arrow_bytes = exported_bytes(g->schema->plan, res->chunks);
    g->arenas[size_t(group)].reset();
    *out = res.release();
    return RV_OK;
}

void rv_gather_free(rv_gather* g) { delete g; }

// CUDA IPC plumbing for the peers' view of the leader's arena (64-byte handles).
rv_status rv_ipc_export(void* dev_ptr, uint8_t* handle64) {
    if (!dev_ptr || !handle64) return fail(RV_ERR_INVALID, "bad argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    cudaIpcMemHandle_t h;
    RV_CUDA(cudaIpcGetMemHandle(&h, dev_ptr));
    std::memcpy(handle64, &h, 64);
    return RV_OK;
}
rv_status rv_ipc_open(const uint8_t* handle64, void** out) {
    if (!handle64 || !out) return fail(RV_ERR_INVALID, "bad argument");
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle64, 64);
    RV_CUDA(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
    return RV_OK;
}
rv_status rv_ipc_close(void* p) {
    if (!p) return RV_OK;
    RV_CUDA(cudaIpcCloseMemHandle(p));
    return RV_OK;
}

}  // extern "C"


// ---- Avro object container files (ocf.hpp) ---------------------------------------------------------------------------
namespace {

// rv_decode_ocf_host, rv_decode_ocf_host_projected when `columns` is not null, rv_decode_ocf_host_resolved when `reader` is
// not null.
rv_status decode_ocf(const uint8_t* file, int64_t len, int64_t num_chunks, const char* const* columns, int64_t n_columns,
                     rv_schema** schema_out, rv_result** out, const rv_schema* reader = nullptr) {
    if (!file || len < 0 || !schema_out || !out) return fail(RV_ERR_INVALID, "null argument");
    *schema_out = nullptr;
    *out = nullptr;
    OcfIndex ix;
    try {
        ix = ocf_index(file, len);
    } catch (const std::exception& e) {
        return fail(RV_ERR_FRAME, e.what());
    }
    rv_schema* s = nullptr;
    rv_status st = rv_schema_parse(ix.schema_json.data(), ix.schema_json.size(), &s);
    if (st) return st;
    rv_schema* file_schema = nullptr;  // resolved: the record offsets are found by walking the file's (the writer's) own plan
    if (reader) {
        st = rv_schema_resolve(s, reader, &file_schema);
        std::swap(s, file_schema);
        if (st) { rv_schema_release(file_schema); return st; }
    }
    struct ReleaseFile { rv_schema* s; ~ReleaseFile() { if (s) rv_schema_release(s); } } rel_file{file_schema};
    if (columns) {
        rv_schema* full = s;
        st = rv_schema_project(full, columns, n_columns, &s);
        rv_schema_release(full);
        if (st) return st;
    }
    struct Release { rv_schema* s; bool armed = true; ~Release() { if (armed) rv_schema_release(s); } } rel{s};
    st = check_decodable(s);
    if (st) return st;
    int device = 0;
    st = ensure_cuda(&device);
    if (st) return st;
    cudaStream_t stream = nullptr;
    const int64_t n = ix.n_records;
    DevBuf d_file, d_blocks, d_off, d_err;
    RV_CUDA(d_file.alloc(size_t(len) + 64, stream));
    RV_CUDA(d_off.alloc(size_t(n + 1) * 8, stream));
    RV_CUDA(d_err.alloc(16, stream));
    SyncOnExit guard{stream};
    RV_CUDA(upload(static_cast<uint8_t*>(d_file.p), file, size_t(len), device, stream));
    if (n > 0) {
        rv_schema* walk_schema = file_schema ? file_schema : s;
        DevicePlan dp;
        st = device_plan(walk_schema, device, &dp);
        if (st) return st;
        std::vector<OcfBlockDev> blocks(ix.blocks.size());
        for (size_t i = 0; i < blocks.size(); ++i) blocks[i] = OcfBlockDev{ix.blocks[i].data_off, ix.blocks[i].size, ix.blocks[i].count, ix.blocks[i].rec_base};
        RV_CUDA(d_blocks.alloc(blocks.size() * sizeof(OcfBlockDev), stream));
        RV_CUDA(cudaMemcpyAsync(d_blocks.p, blocks.data(), blocks.size() * sizeof(OcfBlockDev), cudaMemcpyHostToDevice, stream));
        RV_CUDA(cudaMemsetAsync(d_err.p, 0xFF, 8, stream));
        OcfParams q{};
        q.data = static_cast<const uint8_t*>(d_file.p);
        q.blocks = static_cast<const OcfBlockDev*>(d_blocks.p);
        q.n_blocks = int32_t(blocks.size());
        q.nodes = dp.nodes; q.n_nodes = int32_t(walk_schema->plan.nodes.size());
        q.n_streams = int32_t(walk_schema->plan.streams.size());
        q.sym_off = dp.sym_off; q.sym_bytes = dp.sym_bytes;
        q.offsets = static_cast<int64_t*>(d_off.p);
        q.n_records = n;
        q.end_off = ix.end_off;
        q.err = static_cast<unsigned long long*>(d_err.p);
        launch_ocf_offsets(q, stream);
        RV_CUDA(cudaGetLastError());
        unsigned long long err_word = ~0ull;
        RV_CUDA(cudaMemcpyAsync(&err_word, d_err.p, 8, cudaMemcpyDeviceToHost, stream));
        RV_CUDA(cudaStreamSynchronize(stream));   // (the block table on the host stack is done with as well)
        if (err_word != ~0ull) {
            const uint32_t code = uint32_t(err_word & 0xFF);
            return fail(status_of(code), std::string(err_text(code)) + " (record " + std::to_string(int64_t(err_word >> 8)) + ")");
        }
    }
    try {
        st = decode_on_device(s, static_cast<const uint8_t*>(d_file.p), static_cast<const int64_t*>(d_off.p), n, num_chunks, InputHints{}, stream, device, out);
    } catch (const std::exception& e) {
        st = fail(RV_ERR_INVALID, e.what());
    }
    if (st) return st;
    float ms = 0;
    st = arena_to_host(**out, *(*out)->arenas[0], stream, &ms);
    if (st) { rv_result_free(*out); *out = nullptr; return st; }
    guard.armed = false;
    rel.armed = false;
    *schema_out = s;
    return RV_OK;
}

}  // namespace

extern "C" rv_status rv_decode_ocf_host(const uint8_t* file, int64_t len, int64_t num_chunks, rv_schema** schema_out, rv_result** out) {
    return decode_ocf(file, len, num_chunks, nullptr, 0, schema_out, out);
}

extern "C" rv_status rv_decode_ocf_host_projected(const uint8_t* file, int64_t len, int64_t num_chunks, const char* const* columns,
                                                  int64_t n_columns, rv_schema** schema_out, rv_result** out) {
    if (!columns && n_columns != 0) return fail(RV_ERR_INVALID, "null argument");
    if (!columns) return fail(RV_ERR_INVALID, "column projection: the column list is empty");
    return decode_ocf(file, len, num_chunks, columns, n_columns, schema_out, out);
}

extern "C" rv_status rv_decode_ocf_host_resolved(const uint8_t* file, int64_t len, int64_t num_chunks, const rv_schema* reader,
                                                 const char* const* columns, int64_t n_columns, rv_schema** schema_out, rv_result** out) {
    if (!reader || (!columns && n_columns != 0)) return fail(RV_ERR_INVALID, "null argument");
    return decode_ocf(file, len, num_chunks, columns, n_columns, schema_out, out, reader);
}

extern "C" {

rv_status rv_result_to_host(rv_result* r) {
    if (!r) return fail(RV_ERR_INVALID, "null result");
    float ms = 0;
    for (auto& a : r->arenas) {
        rv_status st = arena_to_host(*r, *a, nullptr, &ms);
        if (st) return st;
    }
    t_timings[5] = ms;
    return RV_OK;
}

rv_status rv_decode_host(const rv_schema* s_, const uint8_t* data, const int64_t* offsets, int64_t n,
                         int64_t num_chunks, rv_result** out) {
    return rv_decode_host_framed(s_, data, offsets, n, num_chunks, nullptr, out);
}

rv_status rv_decode_host_framed(const rv_schema* s_, const uint8_t* data, const int64_t* offsets, int64_t n,
                                int64_t num_chunks, const rv_framing* framing_, rv_result** out) {
    if (!out) return fail(RV_ERR_INVALID, "null argument");
    *out = nullptr;
    rv_schema* s = const_cast<rv_schema*>(s_);
    rv_status st = check_decodable(s);
    if (st) return st;
    st = framing_ok(framing_);
    if (st) return st;
    const rv_framing framing = framing_ ? *framing_ : rv_framing{0, 0, -1};
    if (n < 0 || (n > 0 && (!data || !offsets))) return fail(RV_ERR_INVALID, "bad input pointers");
    int device = 0;
    st = ensure_cuda(&device);
    if (st) return st;
    const int64_t k = clamp_chunks(num_chunks, n);
    float h2d = 0, d2h = 0;
    // pipelining pays when every chunk is big enough to amortise its own launches and copies; many small
    // chunks go through ONE launch that handles all chunks at once
    if (k < 2 || n / k < 16384 || !pipeline_enabled()) {
        st = decode_host_range(s, data, offsets, 0, n, num_chunks, nullptr, device, out, &h2d, &d2h, framing);
        t_timings[4] = h2d;
        t_timings[5] = d2h;
        return st;
    }
    // Chunks are independent batches (deserialize.rs:57-68,92-119): the GPU-side analogue of the reference fanning
    // chunks out to its thread pool.
    const int64_t chunk_rows = n / k;
    struct Call {
        std::mutex mu;
        std::condition_variable cv;
        int64_t left;
        float acc[6] = {0, 0, 0, 0, 0, 0};
        int launches = 0, passes = 0;
        long long slow = 0;
        const char* walker = "none";
        int tile = 0;
    } call;
    call.left = k;
    std::vector<rv_result*> parts(size_t(k), nullptr);
    std::vector<rv_status> status(size_t(k), RV_OK);
    std::vector<std::string> message{size_t(k), std::string()};
    WorkerPool& pool = worker_pool(device);
    for (int64_t i = 0; i < k; ++i) {
        pool.submit([&, i](cudaStream_t stream) {
            const int64_t r0 = i * chunk_rows, r1 = (i == k - 1) ? n : r0 + chunk_rows;
            float hm = 0, dm = 0;
            rv_status rc;
            try {
                rc = decode_host_range(s, data, offsets, r0, r1, 1, stream, device, &parts[size_t(i)], &hm, &dm, framing);
            } catch (const std::exception& e) {
                rc = fail(RV_ERR_INVALID, e.what());
            }
            status[size_t(i)] = rc;
            if (rc) message[size_t(i)] = t_error;
            std::lock_guard<std::mutex> g(call.mu);
            for (int q = 0; q < 4; ++q) call.acc[q] += t_timings[q];
            call.acc[4] += hm;
            call.acc[5] += dm;
            call.launches += t_launches;
            call.passes = std::max(call.passes, t_passes);
            call.slow += t_slow_tiles;
            call.walker = t_walker;
            call.tile = call.tile ? std::min(call.tile, t_tile) : t_tile;
            if (--call.left == 0) call.cv.notify_all();
        });
    }
    {
        std::unique_lock<std::mutex> g(call.mu);
        call.cv.wait(g, [&] { return call.left == 0; });
    }
    for (int q = 0; q < 6; ++q) t_timings[q] = call.acc[q];
    t_launches = call.launches;
    t_passes = call.passes;
    t_slow_tiles = call.slow;
    t_walker = call.walker;
    t_tile = call.tile;
    auto res = std::make_unique<rv_result>();
    res->schema = rv_schema_retain(s);
    rv_status first = RV_OK;
    for (int64_t i = 0; i < k; ++i) {
        if (status[size_t(i)] && !first) { first = status[size_t(i)]; t_error = message[size_t(i)]; }  // first failing chunk wins (:115-119)
    }
    for (int64_t i = 0; i < k; ++i) {
        rv_result* part = parts[size_t(i)];
        if (!part) continue;
        if (!first) {
            res->chunks.push_back(std::move(part->chunks[0]));
            res->arenas.push_back(part->arenas[0]);
            res->arrow_bytes += part->arrow_bytes;
        }
        rv_result_free(part);
    }
    if (first) return first;
    *out = res.release();
    return RV_OK;
}

int64_t rv_result_num_batches(const rv_result* r) { return r ? int64_t(r->chunks.size()) : 0; }
int64_t rv_result_num_rows(const rv_result* r, int64_t batch) {
    if (!r || batch < 0 || batch >= int64_t(r->chunks.size())) return -1;
    return r->chunks[size_t(batch)].rows;
}
int64_t rv_result_arrow_bytes(const rv_result* r) { return r ? r->arrow_bytes : 0; }
int64_t rv_result_buffer_bytes(const rv_result* r) {
    if (!r) return 0;
    int64_t total = 0;
    const Arena* last = nullptr;
    for (auto& a : r->arenas) {
        if (a.get() != last) total += int64_t(a->host ? a->host_bytes : a->bytes);
        last = a.get();
    }
    return total;
}

rv_status rv_result_export(rv_result* r, int64_t batch, struct ArrowArray* out_array, struct ArrowSchema* out_schema) {
    if (!r || !out_array) return fail(RV_ERR_INVALID, "null argument");
    if (batch < 0 || batch >= int64_t(r->chunks.size())) return fail(RV_ERR_INVALID, "batch index out of range");
    if (!r->arenas[size_t(batch)]->host) return fail(RV_ERR_INVALID, "result is device-resident: call rv_result_to_host() or rv_result_export_device()");
    if (out_schema) {
        rv_status st = rv_schema_export_arrow(r->schema, out_schema);
        if (st) return st;
    }
    export_batch(r->schema->plan, r->chunks[size_t(batch)], static_cast<const uint8_t*>(r->arenas[size_t(batch)]->host), r->arenas[size_t(batch)], out_array);
    return RV_OK;
}

rv_status rv_result_export_device(rv_result* r, int64_t batch, struct ArrowDeviceArray* out_array, struct ArrowSchema* out_schema) {
    if (!r || !out_array) return fail(RV_ERR_INVALID, "null argument");
    if (batch < 0 || batch >= int64_t(r->chunks.size())) return fail(RV_ERR_INVALID, "batch index out of range");
    if (!r->arenas[size_t(batch)]->dev) return fail(RV_ERR_INVALID, "result was moved to host memory: use rv_result_export()");
    if (out_schema) {
        rv_status st = rv_schema_export_arrow(r->schema, out_schema);
        if (st) return st;
    }
    export_batch(r->schema->plan, r->chunks[size_t(batch)], static_cast<const uint8_t*>(r->arenas[size_t(batch)]->dev), r->arenas[size_t(batch)], &out_array->array);
    out_array->device_id = r->arenas[size_t(batch)]->device;
    out_array->device_type = ARROW_DEVICE_CUDA;
    out_array->sync_event = nullptr;  // the decode call synchronised its stream before returning
    out_array->reserved[0] = out_array->reserved[1] = out_array->reserved[2] = 0;
    return RV_OK;
}

void rv_result_free(rv_result* r) { delete r; }

void* rv_host_alloc(size_t bytes) {
    size_t actual = 0;
    void* p = pinned().get(bytes, &actual);
    if (!p) {
        t_error = "cudaHostAlloc failed (no CUDA device, or out of pinnable memory)";
        return nullptr;
    }
    std::lock_guard<std::mutex> g(g_host_mu);
    g_host_sizes[p] = actual;
    return p;
}
void rv_host_free(void* p) {
    if (!p) return;
    size_t actual = 0;
    {
        std::lock_guard<std::mutex> g(g_host_mu);
        auto it = g_host_sizes.find(p);
        if (it == g_host_sizes.end()) return;
        actual = it->second;
        g_host_sizes.erase(it);
    }
    pinned().put(p, actual);  // back to the slab cache: re-pinning GiB-sized blocks costs ~100s of ms
}

int rv_last_timings(float* out_ms, int cap) {
    int n = cap < 6 ? cap : 6;
    for (int i = 0; i < n; ++i) out_ms[i] = t_timings[i];
    return n;
}
int rv_last_launch_count(void) { return t_launches; }
int rv_last_passes(void) { return t_passes; }
rv_status rv_dev_rebase_i32(int32_t* d_dst, const int32_t* d_src, int64_t n, int32_t add, void* cuda_stream) {
    if (n < 0 || (n > 0 && (!d_dst || !d_src))) return fail(RV_ERR_INVALID, "bad argument");
    launch_rebase_i32(d_dst, d_src, n, add, static_cast<cudaStream_t>(cuda_stream));
    RV_CUDA(cudaGetLastError());
    return RV_OK;
}

rv_status rv_dev_concat_bits(uint32_t* d_dst_words, int64_t dst_bit, const uint32_t* d_src_words, int64_t nbits, void* cuda_stream) {
    if (nbits < 0 || dst_bit < 0 || (nbits > 0 && (!d_dst_words || !d_src_words))) return fail(RV_ERR_INVALID, "bad argument");
    launch_concat_bits(d_dst_words, dst_bit, d_src_words, nbits, static_cast<cudaStream_t>(cuda_stream));
    RV_CUDA(cudaGetLastError());
    return RV_OK;
}

// used by encode.cu (same library, separate translation unit)
void* rv_internal_dev_get(size_t bytes, int device, size_t* actual) { return devmem().get(bytes, device, actual); }
void rv_internal_dev_put(void* p, size_t actual, int device) { devmem().put(p, actual, device); }
const void* rv_schema_avro_root(const rv_schema* s) { return s ? s->avro.get() : nullptr; }
int rv_schema_is_projection(const rv_schema* s) { return s && (!s->keep.empty() || s->res) ? 1 : 0; }  // (or a resolution)
void rv_set_last_error(const char* msg) { t_error = msg ? msg : ""; }

const char* rv_last_walker(void) { return t_walker; }
int rv_last_tile(void) { return t_tile; }
int rv_schema_max_tile(const rv_schema* s) {
    if (!s || !s->has_plan) return -1;
    return int(s->plan.streams.size()) > kWideStreams ? kWideTile : kBlock;
}
const char* rv_schema_jit_status(const rv_schema* s) {
    if (!s) return "null schema";
    std::lock_guard<std::mutex> g(const_cast<rv_schema*>(s)->mu);
    int device = 0;
    if (cudaGetDevice(&device) != cudaSuccess) (void)cudaGetLastError();
    auto it = s->jit.find({device, kBlock});
    if (it == s->jit.end() || !it->second.tried) it = s->jit.find({device, kWideTile});
    t_error = (it != s->jit.end() && it->second.tried) ? it->second.status : "not attempted yet";
    return t_error.c_str();
}
long long rv_last_slow_tiles(void) { return t_slow_tiles; }
void rv_set_jit_enabled(int enabled) { g_jit_override.store(enabled < 0 ? -1 : (enabled ? 1 : 0)); }
void rv_schema_forget_stats(const rv_schema* s_) {
    rv_schema* s = const_cast<rv_schema*>(s_);
    if (!s) return;
    std::lock_guard<std::mutex> g(s->mu);
    s->stats = SchemaStats();
}

int64_t rv_schema_walker_source(const rv_schema* s, char* buf, size_t cap) {
    if (!s || !s->has_plan) return -1;
    const std::string src = generate_walker_source(s->plan);
    if (buf && cap) {
        const size_t n = std::min(cap - 1, src.size());
        std::memcpy(buf, src.data(), n);
        buf[n] = 0;
    }
    return int64_t(src.size());
}

int64_t rv_schema_kernel_source(const rv_schema* s, int tile, char* buf, size_t cap) {
    if (!s || !s->has_plan || (tile != kBlock && tile != rv_schema_max_tile(s))) return -1;
    const std::string src = generate_kernel_source(s->plan, tile);
    if (buf && cap) {
        const size_t n = std::min(cap - 1, src.size());
        std::memcpy(buf, src.data(), n);
        buf[n] = 0;
    }
    return int64_t(src.size());
}

rv_status rv_schema_precompile(const rv_schema* s, const char* arch) {
    rv_status st = check_decodable(s);
    if (st) return st;
    // the kernel at the plan's largest tile, the one a decode takes whenever its windows allow (choose_tile); a plan of
    // more than eight streams whose windows do not fit two 384-row CTAs compiles its 256-row kernel when first needed
    std::vector<char> cubin;
    std::string log;
    if (!jit_cubin(generate_kernel_source(s->plan, rv_schema_max_tile(s)), arch && *arch ? arch : "sm_90a", &cubin, &log, false)) return fail(RV_ERR_CUDA, "NVRTC: " + log);
    return RV_OK;
}
const char* rv_last_error(void) { return t_error.c_str(); }
const char* rv_version(void) { return "pyruhvro_b200 0.2.0 (sm_90a)"; }

}  // extern "C"
