// ctx.cu — hb_ctx: the C ABI of include/herro_b200.h on top of the kernels in features.cu /
// forward.cu.  Host-side responsibilities: replicate the read store, stage target batches
// (cross-read batching: the reference launches one tiny forward per read, src/features.rs:582,
// SURVEY.md F7), drive the kernel sequence on a stream, and re-assemble per-read segments
// the way consensus() does (src/consensus.rs:86-111,222-226).
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <string>
#include <unordered_map>
#include <vector>

#include <pthread.h>
#include <sched.h>
#include <sys/stat.h>

#include "../../include/herro_b200.h"
#include "common.cuh"
#include "forward.h"
#include "windowing.h"
#include "torchscript.h"

using namespace hb;

namespace {

thread_local std::string g_create_err;
thread_local std::string* t_err_sink = nullptr;
std::atomic<uint64_t> g_ctx_generation{1};  // the launch worker reports into its own string

// allocation accounting (hb_stats.host_allocs / ms_host_alloc): page-locked and device allocations are slow and
// serialise with every other CUDA call of the process, so the steady state must not make any
std::atomic<uint64_t> g_allocs{0}, g_alloc_ns{0}, g_submit_wait_ns{0};
struct AllocScope {
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    const char* kind;
    size_t bytes;
    AllocScope(const char* k, size_t b) : kind(k), bytes(b) {}
    ~AllocScope() {
        const uint64_t ns = (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
        g_allocs.fetch_add(1, std::memory_order_relaxed);
        g_alloc_ns.fetch_add(ns, std::memory_order_relaxed);
        static const bool dbg = getenv("HERRO_B200_DEBUG_ALLOC") != nullptr;
        if (dbg) fprintf(stderr, "[herro_b200 alloc] %s %.1f MB %.2f ms\n", kind, (double)bytes / 1e6, (double)ns * 1e-6);
    }
};

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaStream_t st = nullptr;  // lane regions: grown in stream order from the device's memory pool, because
                                // cudaMalloc/cudaFree synchronise the whole device and would stall the other lanes
    // Grow to hold `bytes`: with 1.5x headroom, or exactly (pre-sizing an idle lane from another lane's sizes).  `keep` copies
    // the contents over (a pre-sized lane's last launch stays replayable / inspectable through the debug taps).
    cudaError_t grow(size_t bytes, bool headroom = true, bool keep = false) {
        if (bytes <= cap) return cudaSuccess;
        const size_t ncap = headroom ? bytes + bytes / 2 + 256 : bytes;
        AllocScope as_(st ? "device(stream-ordered)" : "device", ncap);
        void* np = nullptr;
        cudaError_t e = st ? cudaMallocAsync(&np, ncap, st) : cudaMalloc(&np, ncap);
        if (e != cudaSuccess) return e;
        if (keep && p) { if (st) cudaMemcpyAsync(np, p, cap, cudaMemcpyDeviceToDevice, st); else cudaMemcpy(np, p, cap, cudaMemcpyDeviceToDevice); }
        if (p) { if (st) cudaFreeAsync(p, st); else cudaFree(p); }
        p = np;
        cap = ncap;
        return cudaSuccess;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return (T*)p; }
};

struct PinBuf {
    void* p = nullptr;
    size_t cap = 0;
    // grow to hold `bytes`, with 1.5x headroom or exactly; the contents are not kept
    cudaError_t grow(size_t bytes, bool headroom = true) {
        if (bytes <= cap) return cudaSuccess;
        const size_t ncap = headroom ? bytes + bytes / 2 + 256 : bytes;
        AllocScope as_("pinned(lane)", ncap);
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = cudaMallocHost(&p, ncap);
        if (e == cudaSuccess) cap = ncap;
        return e;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return (T*)p; }
};

// grow-only pinned host array: target batches are staged directly in page-locked memory so the
// launch worker can cudaMemcpyAsync from them without a second copy
template <class T>
struct PinVec {
    T* p = nullptr;
    size_t n = 0, cap = 0;
    int dev = 0;  // device whose context owns the allocation (set before first growth)
    PinVec() {}
    PinVec(const PinVec&) = delete;
    PinVec& operator=(const PinVec&) = delete;
    PinVec(PinVec&& o) noexcept : p(o.p), n(o.n), cap(o.cap), dev(o.dev) { o.p = nullptr; o.n = o.cap = 0; }
    PinVec& operator=(PinVec&& o) noexcept {
        if (this != &o) { release(); p = o.p; n = o.n; cap = o.cap; dev = o.dev; o.p = nullptr; o.n = o.cap = 0; }
        return *this;
    }
    ~PinVec() { release(); }
    void release() { if (p) cudaFreeHost(p); p = nullptr; n = cap = 0; }
    bool reserve(size_t want) {
        if (want <= cap) return true;
        if (want * sizeof(T) > ((size_t)24 << 30)) return false;  // a staging array of > 24 GB is a sizing bug, not a workload: fail, do not pin
        size_t ncap = (n == 0) ? std::max<size_t>(want, 4096) : std::max<size_t>(want * 2, 4096);
        if (ncap * sizeof(T) > ((size_t)24 << 30)) ncap = want;
        AllocScope as_("pinned(staging)", ncap * sizeof(T));
        T* np = nullptr;
        int cur = -1;
        if (cudaGetDevice(&cur) != cudaSuccess || cur != dev) cudaSetDevice(dev);  // growth is rare: only then touch the runtime
        if (cudaHostAlloc((void**)&np, ncap * sizeof(T), cudaHostAllocPortable) != cudaSuccess) return false;
        if (n) memcpy(np, p, n * sizeof(T));
        if (p) cudaFreeHost(p);
        p = np;
        cap = ncap;
        return true;
    }
    bool push_back(const T& v) { if (!reserve(n + 1)) return false; p[n++] = v; return true; }
    bool append(const T* src, size_t k) { if (!reserve(n + k)) return false; if (k) memcpy(p + n, src, k * sizeof(T)); n += k; return true; }
    bool resize(size_t k) { if (!reserve(k)) return false; n = k; return true; }
    size_t size() const { return n; }
    bool empty() const { return n == 0; }
    T* data() { return p; }
    const T* data() const { return p; }
    T& operator[](size_t i) { return p[i]; }
    const T& operator[](size_t i) const { return p[i]; }
    void clear() { n = 0; }
    const T* begin() const { return p; }
    const T* end() const { return p + n; }
};

struct HostBatch {
    PinVec<DevTarget> tgt;
    PinVec<DevWin> win;
    PinVec<DevOverlap> ovl;
    PinVec<DevOW> ow;
    PinVec<uint8_t> cig;
    uint64_t op_cap = 0;      // op slots of host-windowed overlap-windows (assigned here)
    uint64_t raw_cap = 0;     // raw-op slots of device-windowed alignments (cig_len / 2 + 1 each)
    uint64_t dev_op_cap = 0;  // bound on the op slots their overlap-windows need (assigned by a scan on the device)
    uint32_t n_raw = 0;       // device-windowed alignments
    HostBatch() {}
    explicit HostBatch(int dev) { tgt.dev = win.dev = ovl.dev = ow.dev = cig.dev = dev; }
    void clear() { tgt.clear(); win.clear(); ovl.clear(); ow.clear(); cig.clear(); op_cap = raw_cap = dev_op_cap = 0; n_raw = 0; }
};

struct Result {
    uint32_t rid;
    int status;
    std::vector<uint32_t> seg_len;
    std::vector<uint8_t> seq;
    std::string msg;  // why status != HB_OK
};

struct FwdBufs {  // the forward region's arrays besides the work list, which is part of BatchView
    float *logits, *info;
    uint8_t* ws;
};

struct GatherSizes {  // host store: the arrays k_reads_in fills in a launch's batch region; n_reads == 0: the uploaded store
    uint32_t n_reads = 0, n_list = 0;
    uint64_t words = 0, qual = 0;
};

struct LastLaunch {  // host copies of per-window metadata of the most recent launch (debug taps / replay)
    bool valid = false;
    std::vector<DevWin> win;
    std::vector<uint32_t> w_L, w_nsel, w_nsup;
    std::vector<uint64_t> w_rowbase, w_supbase;
    std::vector<uint32_t> ow_qid;  // KEEP_DEBUG: query read of every overlap-window (feature dump)
    std::unordered_map<uint64_t, uint32_t> index;  // (rid << 32 | wid) -> window
    uint64_t n_sup = 0, total_rows = 0;
    // the counts the lane's scratch was carved from, besides those in `view` (a pre-sized lane carves the view again)
    size_t cig_bytes = 0;
    uint64_t op_slots = 0, raw_slots = 0;
    GatherSizes gs;
    BatchView view;
    FwdBufs fwd;
    ReadsInArgs gather{};  // host store: the gather the launch began with (replays run it again)
};

// What one hb_features_batch produced, in the caller's order (targets as given, each target's windows in wid order).  The bulk
// arrays stay in the features lane's regions until hb_features_fetch copies them out.
struct FeatResult {
    bool valid = false;
    hb_features_shape shape{};
    BatchView view;                       // the lane's regions as the call left them
    std::vector<int32_t> status;          // per target
    std::vector<uint32_t> n_windows;
    std::vector<uint32_t> rows, n_sup, n_ids, dev_win;  // per window; dev_win: the window in `view`, ~0u for a failed target
    std::vector<uint8_t> n_alns;
    std::vector<uint64_t> dev_rowbase;    // per window of `view`: its first row in the row arena
    std::vector<uint32_t> batch_B, batch_Lmax, batch_win;
};

}  // namespace

// The read store in host memory (hb_read_store_create): every read's words and qualities in one page-locked block that every
// device of the process can map, each read 16-byte aligned and padded to 16 bytes (zero words, quality 33), so that k_reads_in
// moves whole 16-byte vectors.
struct hb_read_store {
    uint8_t* block = nullptr;                  // cudaHostAlloc(Portable | Mapped): the words of all reads, then their qualities
    uint64_t words_bytes = 0, bytes = 0;
    std::vector<uint64_t> word_off, qual_off;  // per read, in words / bytes from the start of each section
    std::vector<uint32_t> len;
    uint32_t n_reads = 0, max_len = 0;
    std::atomic<uint32_t> attached{0};         // contexts using the store; it must outlive them
};

struct hb_ctx {
    int device = 0;
    hb_options opt{};
    std::string err;
    std::mutex mu;

    // weights
    FwdWeights wt{};
    std::vector<void*> weight_allocs;

    // read store
    bool have_reads = false;
    uint32_t n_reads = 0;
    std::vector<uint32_t> read_len;
    DevBuf d_words, d_word_off, d_len, d_qual, d_qual_off, d_ln;
    uint32_t ln_n = 0;
    ReadStoreView rs{};  // with a host store only len and n: each launch views its gathered reads
    hb_read_store* store = nullptr;  // hb_attach_read_store; nullptr: the uploaded store above
    const uint64_t* store_words = nullptr;  // the store's sections as this device maps them
    const uint8_t* store_qual = nullptr;

    // staging: every submitting (feature) thread fills its own batch without taking the context lock;
    // full batches are handed to the launch worker's queue
    struct ThreadSlot { std::thread::id owner; HostBatch batch; uint32_t handed = 0; /* batches handed over since the last flush */ };
    std::vector<std::unique_ptr<ThreadSlot>> slots;
    PinBuf pin_in;  // staging of hb_upload_reads
    // Launch lanes (stream + device scratch + pinned result buffers each), one worker thread per lane:
    // while lane A's worker does its host work (copy-back, per-read reassembly), lane B's batch keeps the GPU busy.
    struct Lane {
        cudaStream_t stream = nullptr;
        cudaEvent_t ev[8]{};
        KTimer kt;
        // device scratch, one region per moment its size becomes known: the batch (carve_batch), the row arena (carve_rows)
        // and the supported positions (carve_fwd)
        DevBuf d_batch, d_rows, d_fwd;
        PinBuf pin_small, pin_out;  // readback of the counters and per-window metadata (carve_readback), of the emitted bytes
        uint64_t rows_cap = 0;
        uint64_t seen_sizes = 0;  // version of hb_ctx::lane_sizes this lane has been pre-sized to
        LastLaunch last;
        std::thread worker;
        // host store: the read list of the launch being staged, and a stamp per read that marks it listed
        PinVec<ReadCopy> read_list;
        std::vector<uint32_t> stamp;
        uint32_t stamp_gen = 0;
        void release() {
            d_batch.release(); d_rows.release(); d_fwd.release();
            pin_small.release(); pin_out.release();
            read_list.release();
            for (auto& e : ev) if (e) cudaEventDestroy(e);
            kt.destroy();
            if (stream) cudaStreamDestroy(stream);
        }
    };
    // Largest region capacities (and row arena) any lane has needed so far.  A lane that has not run yet (or ran smaller batches)
    // grows its regions to these while it is idle, so that its first real batch allocates nothing (r01: 26 allocations / 226 ms
    // inside the timed region at 8 GPUs, when host contention made the third lane start its first batch there).
    struct LaneSizes { size_t batch = 0, rows = 0, fwd = 0, pin_small = 0, pin_out = 0; uint64_t rows_cap = 0; };
    LaneSizes lane_sizes;
    uint64_t lane_sizes_version = 0;
    static constexpr int MAX_LANES = 4;
    Lane lanes[MAX_LANES];
    int n_lanes = 3;     // HERRO_B200_LANES overrides (1..4)
    uint32_t min_launch = 256;  // smallest per-thread hand-over unless launch_targets itself is smaller (HERRO_B200_MIN_LAUNCH: experiments)
    int last_lane = -1;  // lane of the most recently finished launch (debug taps / replay)
    uint32_t chunk_pos = 65536;  // supported positions per forward pass (HERRO_B200_CHUNK_POS): one pass per launch unless huge
    // hb_forward_batch's lane: its own stream, events, timer and grow-only scratch, which the launch lanes never touch.  Calls
    // serialise on its mutex.
    struct FwdLane {
        std::mutex mu;
        cudaStream_t stream = nullptr;
        cudaEvent_t ev[3]{};  // the caller's stream, forward start, forward end
        KTimer kt;
        PinBuf pin_in, pin_out;     // input region (carve_fwd_in) + the work list; the host outputs
        DevBuf d_in, d_mat, d_fwd;  // input region; the [rows][32] matrices; the forward region (carve_fwd)
        void release() {
            d_in.release(); d_mat.release(); d_fwd.release();
            pin_in.release(); pin_out.release();
            for (auto& e : ev) if (e) cudaEventDestroy(e);
            kt.destroy();
            if (stream) cudaStreamDestroy(stream);
        }
    } fwd;
    // hb_consensus_batch's lane, shaped like the forward lane, so that a host can run the consensus of one read while the
    // forward of the next one runs.  Calls serialise on its mutex.
    struct ConsLane {
        std::mutex mu;
        cudaStream_t stream = nullptr;
        cudaEvent_t ev[3]{};     // the caller's stream, consensus start, consensus end
        KTimer kt;
        PinBuf pin_in, pin_out;  // input region (carve_cons_in); the emitted lengths and bytes
        DevBuf d_in, d_out;      // input region; the consensus region (carve_cons_out)
        std::vector<uint32_t> order;       // host scratch: key sorting
        std::vector<uint8_t> seq;          // the segments before they are copied out
        std::vector<uint32_t> seg_len;
        void release() {
            d_in.release(); d_out.release();
            pin_in.release(); pin_out.release();
            for (auto& e : ev) if (e) cudaEventDestroy(e);
            kt.destroy();
            if (stream) cudaStreamDestroy(stream);
        }
    } cons;
    // hb_features_batch's lane: a launch lane that no worker owns (stream, events, timer, batch and row regions) and never publishes
    // its sizes to the pipeline's lanes, its own staging batch, and the tables and staging of hb_features_fetch.  Calls of
    // hb_features_batch and hb_features_fetch serialise on its mutex.
    struct FeatLane {
        std::mutex mu;
        Lane lane;
        HostBatch hbt;
        PinBuf pin_n1, pin_tab;  // the windows' surviving-overlap counts; the output tables, staged for one copy
        DevBuf d_tab, d_out;     // the output tables; the host-bound outputs before their copy
        FeatResult res;
        uint64_t ticket = 0;
        void release() {
            lane.release();
            pin_n1.release(); pin_tab.release();
            d_tab.release(); d_out.release();
            hbt = HostBatch();
        }
    } feat;
    bool no_model = false;  // HB_FLAG_NO_MODEL: no weights; the calls that run the forward refuse

    std::deque<Result> results;
    hb_stats stats{};

    // launch worker: batches are processed asynchronously so that the host can stage batch i+1
    // (and drain results of batch i-1) while batch i is on the GPU
    std::condition_variable cv_work, cv_idle;
    std::deque<HostBatch> queue;
    std::vector<HostBatch> pool;  // recycled staging batches (keep their pinned capacity)
    bool stop = false;
    int busy = 0;  // lanes currently inside a launch
    int worker_rc = HB_OK;
    std::string worker_err;
    bool idle() const { return queue.empty() && busy == 0; }
    size_t cap_hint[5] = {0, 0, 0, 0, 0};  // largest batch array sizes seen (tgt, win, ovl, ow, cig)
    std::atomic<uint32_t> handed_total{0};  // batches handed over by all threads since the last flush (slow-start ramp)
    std::atomic<uint32_t> n_slots{0};       // submitting threads registered since the last flush
    std::atomic<bool> time_kernels{false};  // hb_set_kernel_timing
    uint64_t alloc_base[3] = {0, 0, 0};     // g_allocs / g_alloc_ns / g_submit_wait_ns at the last hb_reset_stats
    uint64_t generation = 0;  // distinguishes contexts that reuse an address (thread-local slot cache)
    // debugging aids read from the environment once, in hb_create
    bool host_windowing = false;     // HERRO_B200_HOST_WINDOWING: hb_submit_alignments runs extract_windows on the host (A-B test)
    bool pileup_v1 = false;          // HERRO_B200_PILEUP_V1: the former position-walk pileup kernel (A-B parity test)
    uint32_t arena_rows_per_win = 0; // HERRO_B200_ARENA_ROWS: initial row-arena rows per window (default 1.5 W); tests shrink it
                                     // to force the overflow -> regrow -> relaunch path
    // staging-batch pool: every HostBatch that exists is counted, so the steady state allocates nothing
    uint32_t batches_alive = 0;
    // CPUs of the NUMA node the GPU hangs off (empty: unknown); launch workers are bound to them, hb_bind_calling_thread
    // does the same for the host's feature / consumer threads
    cpu_set_t node_cpus;
    bool have_node_cpus = false;
    int numa_node = -1;
};

namespace {

std::string& errref(hb_ctx* ctx) { return t_err_sink ? *t_err_sink : ctx->err; }

#define CK(call)                                                                      \
    do {                                                                              \
        cudaError_t e__ = (call);                                                     \
        if (e__ != cudaSuccess) {                                                     \
            errref(ctx) = std::string(#call) + ": " + cudaGetErrorString(e__);        \
            return HB_ERR_CUDA;                                                       \
        }                                                                             \
    } while (0)

int fail(hb_ctx* ctx, int code, const std::string& msg) {
    errref(ctx) = msg;
    return code;
}

// ---------------------------------------------------------------------------------- weights
#pragma pack(push, 1)
struct BlobHeader {
    char magic[8];
    uint32_t version, n_tensors;
    uint32_t cfg[16];
};
struct BlobEntry {
    char name[48];
    uint32_t dtype, ndim, shape[4];
    uint64_t offset, nbytes;
};
#pragma pack(pop)

// NUMA node of the GPU (sysfs) and that node's CPU list: ranks sharing a box must not pile their host threads onto one socket
void probe_numa(hb_ctx* ctx) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, (int)sizeof bus, ctx->device) != cudaSuccess) return;
    for (char* c = bus; *c; c++) *c = (char)tolower(*c);
    std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
    FILE* f = fopen(path.c_str(), "r");
    if (!f) return;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return;
    path = "/sys/devices/system/node/node" + std::to_string(node) + "/cpulist";
    f = fopen(path.c_str(), "r");
    if (!f) return;
    char line[4096] = {0};
    const bool got = fgets(line, sizeof line, f) != nullptr;
    fclose(f);
    if (!got) return;
    cpu_set_t allowed, set;
    CPU_ZERO(&set);
    if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return;
    int n = 0;
    for (const char* p = line; *p;) {  // "0-31,64-95"
        char* e;
        long a = strtol(p, &e, 10), b2 = a;
        if (e == p) break;
        if (*e == '-') { p = e + 1; b2 = strtol(p, &e, 10); }
        for (long c = a; c <= b2 && c < CPU_SETSIZE; c++)
            if (CPU_ISSET((int)c, &allowed)) { CPU_SET((int)c, &set); n++; }
        p = (*e == ',') ? e + 1 : e;
        if (*e != ',') break;
    }
    if (n == 0) return;
    ctx->node_cpus = set;
    ctx->have_node_cpus = true;
    ctx->numa_node = node;
}

// A model file as the canonical tensor table (names and forms of herro_b200/weights.py): either the HB200W1 blob, or a
// TorchScript archive of the same architecture - what the reference's `-m` names (src/inference.rs:185) - read by torchscript.cpp.
struct ModelFile {
    uint32_t cfg[13] = {0};  // tokens, emb, reads, stem_k, C, H, layers, F, D, classes, pos_layers, pos_heads, pos_ffn
    std::map<std::string, std::vector<float>> T;
};
int read_model_file(const char* path, ModelFile& mf, std::string& err) {
    FILE* f = fopen(path, "rb");
    if (!f) { err = std::string("cannot open model file ") + path; return HB_ERR_MODEL; }
    fseek(f, 0, SEEK_END);
    long sz = ftell(f);
    fseek(f, 0, SEEK_SET);
    if (sz < 0) { fclose(f); err = "cannot size model file"; return HB_ERR_MODEL; }
    std::vector<uint8_t> buf((size_t)sz);
    if (fread(buf.data(), 1, (size_t)sz, f) != (size_t)sz) { fclose(f); err = "short read on model file"; return HB_ERR_MODEL; }
    fclose(f);
    if (ts_is_zip(buf.data(), buf.size())) {
        TsModel m;
        if (!ts_read_archive(buf.data(), buf.size(), m)) { err = "TorchScript archive: " + m.err; return HB_ERR_MODEL; }
        TsDims d;
        if (!ts_to_canonical(m, 4, d, mf.T, err)) { err = "TorchScript archive: " + err; return HB_ERR_MODEL; }
        const uint32_t c[13] = {12, 6, 31, (uint32_t)d.stem_k, (uint32_t)d.channels, (uint32_t)d.heads, (uint32_t)d.layers, (uint32_t)d.ffn, (uint32_t)d.collapse, 5,
                                (uint32_t)d.pos_layers, (uint32_t)d.pos_heads, (uint32_t)d.pos_ffn};
        memcpy(mf.cfg, c, sizeof c);
        return HB_OK;
    }
    if ((size_t)sz < sizeof(BlobHeader)) { err = "model file too small"; return HB_ERR_MODEL; }
    BlobHeader h;
    memcpy(&h, buf.data(), sizeof h);
    // VERSION 2 marks a blob with a position-axis stage (header words 10-12), so that a library without it refuses the file
    if (memcmp(h.magic, "HB200W1\0", 8) != 0 || (h.version != 1 && h.version != 2)) {
        err = "neither an HB200W1 weights blob nor a TorchScript archive";
        return HB_ERR_MODEL;
    }
    memcpy(mf.cfg, h.cfg, sizeof mf.cfg);
    for (uint32_t i = 0; i < h.n_tensors; i++) {
        BlobEntry e;
        size_t eo = sizeof(BlobHeader) + (size_t)i * sizeof(BlobEntry);
        if (eo + sizeof e > (size_t)sz) { err = "truncated tensor table"; return HB_ERR_MODEL; }
        memcpy(&e, buf.data() + eo, sizeof e);
        if (e.dtype != 0 || e.offset > (uint64_t)sz || e.nbytes > (uint64_t)sz - e.offset || (e.offset & 3u) || (e.nbytes & 3u)) {
            err = "bad tensor entry";
            return HB_ERR_MODEL;
        }
        char nm[49];
        memcpy(nm, e.name, 48);
        nm[48] = 0;
        std::vector<float>& v = mf.T[nm];
        v.resize((size_t)(e.nbytes / 4));
        memcpy(v.data(), buf.data() + e.offset, (size_t)e.nbytes);
    }
    return HB_OK;
}

int load_weights(hb_ctx* ctx, const char* path) {
    ModelFile mf;
    {
        std::string e;
        const int rc = read_model_file(path, mf, e);
        if (rc != HB_OK) return fail(ctx, rc, e);
    }
    const uint32_t* cfg = mf.cfg;
    if (cfg[0] != 12 || cfg[1] != 6 || cfg[2] != 31 || cfg[9] != 5)
        return fail(ctx, HB_ERR_MODEL, "unsupported fixed dimensions (tokens/emb/reads/classes)");
    FwdWeights& wt = ctx->wt;
    wt.stem_k = (int)cfg[3]; wt.C = (int)cfg[4]; wt.H = (int)cfg[5]; wt.layers = (int)cfg[6];
    wt.F = (int)cfg[7]; wt.D = (int)cfg[8];
    if (wt.layers < 1 || wt.layers > MAX_LAYERS || wt.H < 1 || wt.C % wt.H || (wt.C / wt.H != 16 && wt.C / wt.H != 32) ||
        wt.C % 128 || wt.F % 128 || wt.D % 128 || !(wt.stem_k & 1) || wt.stem_k > 129 || wt.C > 1024)
        return fail(ctx, HB_ERR_MODEL, "unsupported model dimensions (need C,F,D % 128 == 0, head_dim 16 or 32, odd stem_k)");
    wt.pos_layers = (int)cfg[10]; wt.pos_heads = (int)cfg[11]; wt.pos_ffn = (int)cfg[12];
    if (wt.pos_layers) {
        if (wt.pos_layers > MAX_LAYERS)
            return fail(ctx, HB_ERR_MODEL, "unsupported pos_layers " + std::to_string(wt.pos_layers) + " (at most " + std::to_string(MAX_LAYERS) + ")");
        if (wt.pos_heads < 1 || wt.D % wt.pos_heads || (wt.D / wt.pos_heads != 32 && wt.D / wt.pos_heads != 64))
            return fail(ctx, HB_ERR_MODEL, "unsupported pos_heads " + std::to_string(wt.pos_heads) + " (collapse / pos_heads must be 32 or 64)");
        if (wt.pos_ffn < 128 || wt.pos_ffn % 128)
            return fail(ctx, HB_ERR_MODEL, "unsupported pos_ffn " + std::to_string(wt.pos_ffn) + " (must be a positive multiple of 128)");
    }
    std::unordered_map<std::string, std::pair<const float*, size_t>> T;
    for (auto& kv : mf.T) T[kv.first] = {kv.second.data(), kv.second.size()};
    auto need = [&](const std::string& n, size_t count, const float*& hostp) -> bool {
        auto it = T.find(n);
        if (it == T.end() || it->second.second != count) { ctx->err = "missing/mis-sized tensor " + n; return false; }
        hostp = it->second.first;
        return true;
    };
    auto upload = [&](const float* hostp, size_t count, const float*& devp) -> bool {
        void* d = nullptr;
        if (cudaMalloc(&d, count * 4) != cudaSuccess) { ctx->err = "cudaMalloc(weights)"; return false; }
        ctx->weight_allocs.push_back(d);
        if (cudaMemcpy(d, hostp, count * 4, cudaMemcpyHostToDevice) != cudaSuccess) { ctx->err = "cudaMemcpy(weights)"; return false; }
        devp = (const float*)d;
        return true;
    };
    auto get = [&](const std::string& n, size_t count, const float*& devp) -> bool {
        const float* hp;
        return need(n, count, hp) && upload(hp, count, devp);
    };
    const int C = wt.C, K = wt.stem_k, F = wt.F, D = wt.D;
    const float *emb, *stem_w;
    if (!need("emb", 12 * 6, emb) || !need("stem_w", (size_t)C * 7 * K, stem_w)) return HB_ERR_MODEL;
    // fold the embedding into the conv: tab[j][t][c] = sum_e stem_w[c][e][j] * emb[t][e]
    std::vector<float> tab((size_t)K * 12 * C), wq((size_t)K * C);
    for (int j = 0; j < K; j++)
        for (int c = 0; c < C; c++) {
            for (int t = 0; t < 12; t++) {
                float acc = 0.f;  // fp32, e ascending: the order a direct conv over 7 input channels would use
                for (int e = 0; e < 6; e++) acc = fmaf(stem_w[((size_t)c * 7 + e) * K + j], emb[t * 6 + e], acc);
                tab[((size_t)j * 12 + t) * C + c] = acc;
            }
            wq[(size_t)j * C + c] = stem_w[((size_t)c * 7 + 6) * K + j];
        }
    if (!upload(tab.data(), tab.size(), wt.stem_tab) || !upload(wq.data(), wq.size(), wt.stem_wq)) return HB_ERR_CUDA;
    bool ok = get("stem_b", C, wt.stem_b) && get("read_pos", 31 * (size_t)C, wt.read_pos);
    for (int l = 0; ok && l < wt.layers; l++) {
        const std::string p = "l" + std::to_string(l) + ".";
        FwdLayer& ly = wt.layer[l];
        ok = get(p + "ln1_g", C, ly.ln1_g) && get(p + "ln1_b", C, ly.ln1_b) && get(p + "wqkv", (size_t)3 * C * C, ly.wqkv) &&
             get(p + "bqkv", 3 * (size_t)C, ly.bqkv) && get(p + "wo", (size_t)C * C, ly.wo) && get(p + "bo", C, ly.bo) &&
             get(p + "ln2_g", C, ly.ln2_g) && get(p + "ln2_b", C, ly.ln2_b) && get(p + "w1", (size_t)F * C, ly.w1) &&
             get(p + "b1", F, ly.b1) && get(p + "w2", (size_t)C * F, ly.w2) && get(p + "b2", C, ly.b2);
    }
    ok = ok && get("lnf_g", C, wt.lnf_g) && get("lnf_b", C, wt.lnf_b) && get("wc", (size_t)D * 31 * C, wt.wc) &&
         get("bc", D, wt.bc) && get("wb", 5 * (size_t)D, wt.wb) && get("bb", 5, wt.bb) && get("wi", D, wt.wi) &&
         get("bi", 1, wt.bi);
    const size_t P = (size_t)wt.pos_ffn;
    std::vector<const float*> pos_w(4 * (size_t)wt.pos_layers);  // wqkv, wo, w1, w2 of each position layer (device, fp32)
    for (int l = 0; ok && l < wt.pos_layers; l++) {
        const std::string p = "p" + std::to_string(l) + ".";
        PosLayer& ly = wt.pos[l];
        const float** w4 = &pos_w[4 * (size_t)l];
        ok = get(p + "ln1_g", D, ly.ln1_g) && get(p + "ln1_b", D, ly.ln1_b) && get(p + "wqkv", (size_t)3 * D * D, w4[0]) &&
             get(p + "bqkv", 3 * (size_t)D, ly.bqkv) && get(p + "wo", (size_t)D * D, w4[1]) && get(p + "bo", D, ly.bo) &&
             get(p + "ln2_g", D, ly.ln2_g) && get(p + "ln2_b", D, ly.ln2_b) && get(p + "w1", P * D, w4[2]) &&
             get(p + "b1", P, ly.b1) && get(p + "w2", (size_t)D * P, w4[3]) && get(p + "b2", D, ly.b2);
    }
    if (!ok) return ctx->err.rfind("cuda", 0) == 0 ? HB_ERR_CUDA : HB_ERR_MODEL;
    // bf16 hi/lo split of the contraction weights for the wgmma path (gemm_tc.cu)
    if (cudaDeviceGetAttribute(&wt.num_sms, cudaDevAttrMultiProcessorCount, ctx->device) != cudaSuccess) wt.num_sms = 132;
    auto split = [&](const float* w, size_t n, SplitW& s) -> bool {
        void *hi = nullptr, *lo = nullptr;
        if (split_weights(w, n, &hi, &lo) != cudaSuccess) { ctx->err = "cuda: weight split failed"; return false; }
        ctx->weight_allocs.push_back(hi);
        ctx->weight_allocs.push_back(lo);
        s.hi = hi; s.lo = lo;
        return true;
    };
    for (int l = 0; l < wt.layers; l++) {
        FwdLayer& ly = wt.layer[l];
        if (!split(ly.wqkv, (size_t)3 * C * C, ly.s_qkv) || !split(ly.wo, (size_t)C * C, ly.s_o) ||
            !split(ly.w1, (size_t)F * C, ly.s_1) || !split(ly.w2, (size_t)C * F, ly.s_2)) return HB_ERR_CUDA;
    }
    if (!split(wt.wc, (size_t)D * 31 * C, wt.s_c)) return HB_ERR_CUDA;
    for (int l = 0; l < wt.pos_layers; l++) {
        PosLayer& ly = wt.pos[l];
        const float* const* w4 = &pos_w[4 * (size_t)l];
        if (!split(w4[0], (size_t)3 * D * D, ly.s_qkv) || !split(w4[1], (size_t)D * D, ly.s_o) || !split(w4[2], P * D, ly.s_1) ||
            !split(w4[3], (size_t)D * P, ly.s_2)) return HB_ERR_CUDA;
    }
    // head-grouped copy of Wqkv / bqkv for the fused QKV+attention kernel: row (h, s, d) = row s*C + h*32 + d (s = q,k,v)
    if (C == 128 && wt.H == 4) {
        for (int l = 0; l < wt.layers; l++) {
            const std::string p = "l" + std::to_string(l) + ".";
            const float *hw, *hbias;
            if (!need(p + "wqkv", (size_t)3 * C * C, hw) || !need(p + "bqkv", 3 * (size_t)C, hbias)) return HB_ERR_MODEL;
            std::vector<float> wp((size_t)3 * C * C), bp((size_t)3 * C);
            for (int h = 0; h < 4; h++)
                for (int sI = 0; sI < 3; sI++)
                    for (int d = 0; d < 32; d++) {
                        const size_t dst = (size_t)h * 96 + sI * 32 + d, src = (size_t)sI * C + h * 32 + d;
                        memcpy(&wp[dst * C], hw + src * C, (size_t)C * 4);
                        bp[dst] = hbias[src];
                    }
            const float* dwp = nullptr;
            if (!upload(wp.data(), wp.size(), dwp) || !upload(bp.data(), bp.size(), wt.layer[l].bqkvp)) return HB_ERR_CUDA;
            if (!split(dwp, wp.size(), wt.layer[l].s_qkvp)) return HB_ERR_CUDA;
        }
    }
    // W' of the tensor-core stem: [C][taps*16] = tab of tokens 0..10, wq twice (q_hi, q_lo columns), tab of the pad token 11
    // (the batch-padding rows carry it, and a model's emb[11] need not be zero), zero padding
    wt.stem_kblocks = 0;
    if (C == 128 && K <= 64 && !getenv("HERRO_B200_STEM_SIMT")) {
        const int kbl = (K * 16 + 63) / 64, Kp = kbl * 64;
        std::vector<float> wp((size_t)C * Kp, 0.f);
        for (int c = 0; c < C; c++)
            for (int j = 0; j < K; j++) {
                for (int t = 0; t < 11; t++) wp[(size_t)c * Kp + j * 16 + t] = tab[((size_t)j * 12 + t) * C + c];
                wp[(size_t)c * Kp + j * 16 + 11] = wq[(size_t)j * C + c];
                wp[(size_t)c * Kp + j * 16 + 12] = wq[(size_t)j * C + c];
                wp[(size_t)c * Kp + j * 16 + 13] = tab[((size_t)j * 12 + 11) * C + c];
            }
        const float* dwp = nullptr;
        if (!upload(wp.data(), wp.size(), dwp)) return HB_ERR_CUDA;
        if (!split(dwp, wp.size(), wt.s_stem)) return HB_ERR_CUDA;
        wt.stem_kblocks = kbl;
    }
    if (cudaDeviceSynchronize() != cudaSuccess) { ctx->err = "cuda: weight split kernel failed"; return HB_ERR_CUDA; }
    return HB_OK;
}

// ---------------------------------------------------------------------------------- batch run
template <class T>
size_t vbytes(const PinVec<T>& v) { return v.size() * sizeof(T); }

// A lane's scratch regions are carved the way forward.cu carves the forward workspace: every array starts 256-byte aligned and
// the layout depends only on the counts, so a dry run (base == nullptr) gives a region's size, and carving the same counts
// again after the region moved with its contents gives the same offsets.
struct Carve {
    uint8_t* base;
    size_t bytes = 0;
    template <class T> void operator()(T*& p, size_t n) { p = (T*)(base + bytes); bytes += al256(n * sizeof(T)); }
};

// Batch region, sized from the HostBatch when a launch starts (the view's n_tgt / n_win / n_ovl / n_ow and W, and the CIGAR
// bytes and op slots): inputs, raw and tokenised ops, everything per overlap-window, overlap, window and target, counters.  With a
// host store also the launch's gathered reads, their read list and the offset tables, which become the view's read store.
size_t carve_batch(BatchView& b, size_t cig_bytes, uint64_t op_slots, uint64_t raw_slots, const GatherSizes& gs, ReadsInArgs& g,
                   uint8_t* base) {
    const size_t nt = b.n_tgt, nw = b.n_win, no1 = std::max<size_t>(b.n_ovl, 1), ow1 = std::max<size_t>(b.n_ow, 1);
    const size_t ops = std::max<uint64_t>(op_slots, 1), raw = std::max<uint64_t>(raw_slots, 1);
    Carve c{base};
    c(b.tgt, nt);
    c(b.win, nw);
    c(b.ovl, no1);
    c(b.ow_mut, ow1);
    b.ow = b.ow_mut;
    c(b.cig, std::max<size_t>(cig_bytes, 16));
    c(b.raw_kl, raw);
    c(b.raw_t, raw);
    c(b.raw_q, raw);
    c(b.op_kl, ops);
    c(b.op_t, ops);
    c(b.op_q, ops);
    c(b.ow_nops, ow1);
    c(b.ow_flags, ow1);
    c(b.ow_acc, ow1);
    c(b.ow_tend, ow1);
    c(b.col_ow, ow1);
    c(b.big_key, ow1);
    c(b.big_cand, ow1);
    c(b.big_score, ow1);
    c(b.ow_opoff, ow1);
    c(b.rank_ow, ow1);
    c(b.ovl_n, no1);
    c(b.ovl_tot, no1);
    c(b.ovl_score, no1);
    c(b.aln_nops, no1);
    c(b.aln_flags, no1);
    c(b.w_n1, nw);
    c(b.w_S, nw);
    c(b.sel_ow, nw * TOP_K);
    c(b.w_nsel, nw);
    c(b.rowmap, nw * (size_t)(b.W + 1));
    c(b.w_L, nw);
    c(b.w_rowbase, nw);
    c(b.w_nsup, nw);
    c(b.w_reflmax, nw);
    c(b.w_supbase, nw);
    c(b.w_outlen, nw);
    c(b.w_outoff, nw);
    c(b.tgt_err, nt);
    c(b.counters, CNT_N);
    if (gs.n_reads) {
        c(g.list, gs.n_list);
        c(g.words, READS_FRONT_WORDS + gs.words + READS_BACK_WORDS);
        c(g.qual, READS_FRONT_QUAL + gs.qual + READS_BACK_QUAL);
        c(g.word_off, (size_t)gs.n_reads + 1);
        c(g.qual_off, (size_t)gs.n_reads + 1);
        g.n = gs.n_list;
        g.n_words = gs.words;
        g.n_qual = gs.qual;
        b.rs.words = g.words + READS_FRONT_WORDS;
        b.rs.word_off = g.word_off;
        b.rs.qual = g.qual + READS_FRONT_QUAL;
        b.rs.qual_off = g.qual_off;
    }
    return c.bytes;
}

// Row region, sized from the row arena (the view's rows_cap)
size_t carve_rows(BatchView& b, uint8_t* base) {
    const size_t rows = b.rows_cap;
    Carve c{base};
    c(b.mat_bases, rows * ROW_BYTES);
    c(b.mat_quals, rows * ROW_BYTES);
    c(b.row_emit, rows);
    c(b.sup_row, rows);
    c(b.sup_pk, rows);
    c(b.out_bytes, rows);
    return c.bytes;
}

// Forward region, sized from the supported positions once the first wait has counted them: the work list, the logits and
// the workspace of one forward pass.  A pass holds whole windows (launch_tail), so it is sized for chunk_pos positions or
// the largest window, whichever is larger.
size_t carve_fwd(const hb_ctx* ctx, BatchView& b, FwdBufs& f, uint64_t n_sup, uint32_t max_nsup, uint8_t* base) {
    const size_t n = std::max<uint64_t>(n_sup, 1);
    Carve c{base};
    c(b.fwd_win, n);
    c(b.fwd_row, n);
    c(f.logits, n * 5);
    c(f.info, n);
    c(f.ws, fwd_workspace_bytes(ctx->wt, (uint32_t)std::min<uint64_t>(std::max(ctx->chunk_pos, max_nsup), n)));
    return c.bytes;
}

// Pinned readback of a launch: counters, then per window and per target what the per-read reassembly needs
struct Readback {
    uint32_t *cnt, *outlen, *nsel, *L, *nsup, *terr, *sel;
};
size_t carve_readback(Readback& h, size_t nt, size_t nw, uint8_t* base) {
    Carve c{base};
    c(h.cnt, CNT_N);
    c(h.outlen, nw);
    c(h.nsel, nw);
    c(h.L, nw);
    c(h.nsup, nw);
    c(h.terr, nt);
    c(h.sel, nw * TOP_K);
    return c.bytes;
}

// The counts of a launch and the context's read store (with a host store, carve_batch points it at the gathered reads); the scratch
// pointers are carved from the lane's regions.
BatchView make_view(hb_ctx* ctx, const HostBatch& hbt) {
    BatchView b{};
    b.rs = ctx->rs;
    b.ln_table = ctx->d_ln.as<double>();
    b.ln_table_n = ctx->ln_n;
    b.W = ctx->opt.window_size;
    b.n_tgt = (uint32_t)hbt.tgt.size();
    b.n_win = (uint32_t)hbt.win.size();
    b.n_ovl = (uint32_t)hbt.ovl.size();
    b.n_ow = (uint32_t)hbt.ow.size();
    b.batch_size = ctx->opt.batch_size;
    b.n_raw = hbt.n_raw;
    b.op_base_dev = (uint32_t)hbt.op_cap;
    return b;
}

// Point the view at a row arena of at least `rows` rows, growing the row region if needed.  Its contents are not kept: every
// attempt of a launch fills the row region anew.
int set_rows(hb_ctx* ctx, hb_ctx::Lane* L, BatchView& b, uint64_t rows) {
    if (rows > L->rows_cap) {
        b.rows_cap = rows;
        CK(L->d_rows.grow(carve_rows(b, nullptr)));
        L->rows_cap = rows;
    }
    b.rows_cap = L->rows_cap;
    carve_rows(b, L->d_rows.as<uint8_t>());
    return HB_OK;
}

int zero_scratch(hb_ctx* ctx, hb_ctx::Lane* L, const BatchView& b) {
    CK(cudaMemsetAsync(b.ovl_n, 0, std::max<size_t>(b.n_ovl, 1) * 4, L->stream));
    CK(cudaMemsetAsync(b.ovl_tot, 0, std::max<size_t>(b.n_ovl, 1) * 4, L->stream));
    CK(cudaMemsetAsync(b.tgt_err, 0, (size_t)b.n_tgt * 4, L->stream));
    CK(cudaMemsetAsync(b.counters, 0, CNT_N * 4, L->stream));
    return HB_OK;
}

// The forward over the work list of windows [0, nw) (nsup[nw] positions each, back to back).  A forward pass takes as many whole
// windows as fit in chunk_pos positions; a window larger than that is a pass of its own.  Returns the kernel launches.
uint64_t launch_forward_passes(const hb_ctx* ctx, const BatchView& b, const FwdBufs& f, const uint32_t* nsup, size_t nw, cudaStream_t st,
                               KTimer& kt) {
    uint64_t n0 = 0, launches = 0;
    for (size_t w0 = 0; w0 < nw;) {
        uint64_t np = nsup[w0];
        size_t w1 = w0 + 1;
        while (w1 < nw && np + nsup[w1] <= ctx->chunk_pos) np += nsup[w1++];
        if (np) launches += launch_forward_chunk(b, ctx->wt, (uint32_t)n0, (uint32_t)np, (uint32_t)w0, (uint32_t)(w1 - w0), f.ws, f.logits,
                                                 f.info, st, kt);
        n0 += np;
        w0 = w1;
    }
    return launches;
}

// Algorithmic FLOPs of the forward at n_sup positions in windows of nsup[nw] positions
void add_forward_flops(const hb_ctx* ctx, hb_stats& S, uint64_t n_sup, const uint32_t* nsup, size_t nw) {
    uint64_t gf = 0;
    const uint64_t ff = forward_flops_per_pos(ctx->wt, &gf);
    S.forward_flops += ff * n_sup;
    S.gemm_flops += gf * n_sup;
    uint64_t cf[16];
    forward_class_flops_per_pos(ctx->wt, cf);
    for (int i = 0; i < HB_NUM_KERNEL_CLASSES; i++) S.class_flops[i] += cf[i] * n_sup;
    const uint64_t pa = pos_attn_flops(ctx->wt, nsup, nw);
    S.class_flops[K_POS_ATTN] += pa;
    S.forward_flops += pa;
}

// The forward + consensus part once the supported positions of every window (nsup[nw]) are known.
int launch_tail(hb_ctx* ctx, hb_ctx::Lane* L, const BatchView& b, const FwdBufs& f, const uint32_t* nsup, size_t nw, uint64_t* launches) {
    *launches += launch_features_c2(b, L->stream, L->kt);
    *launches += launch_forward_passes(ctx, b, f, nsup, nw, L->stream, L->kt);
    CK(cudaEventRecord(L->ev[4], L->stream));
    *launches += launch_consensus(b, L->stream, L->kt);
    CK(cudaEventRecord(L->ev[5], L->stream));
    return HB_OK;
}

static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// The segments of one read from its windows' emitted bytes, which lie back to back at `bytes` (src/consensus.rs:90-111,222-226):
// the windows with n_alns >= 2 are concatenated, any other window ends the current segment, and an empty segment is never
// emitted.  (Trimming the read to its first and last window with n_alns >= 2 changes nothing here: the windows outside that
// range only end an empty segment.)  Appends to seq / seg_len; returns the bytes consumed.
uint64_t append_segments(const uint32_t* nsel, const uint32_t* outlen, size_t nw, const uint8_t* bytes, std::vector<uint8_t>& seq,
                         std::vector<uint32_t>& seg_len) {
    uint64_t o = 0;
    size_t start = seq.size();
    for (size_t w = 0; w < nw; w++) {
        if (nsel[w] >= 2) {
            seq.insert(seq.end(), bytes + o, bytes + o + outlen[w]);
        } else if (seq.size() > start) {
            seg_len.push_back((uint32_t)(seq.size() - start));
            start = seq.size();
        }
        o += outlen[w];
    }
    if (seq.size() > start) seg_len.push_back((uint32_t)(seq.size() - start));
    return o;
}

#define SYNC_TIMED() do { const double t__ = now_ms(); CK(cudaStreamSynchronize(L->stream)); t_wait += now_ms() - t__; } while (0)
#define PHASE(i) do { const double t__ = now_ms(); S.ms_worker_phase[i] += t__ - t_mark; t_mark = t__; } while (0)

// Host store: the distinct reads of a staged batch (its targets and every query), each listed once in L->read_list with its place
// in the store and in the batch region, reads laid out in order of first appearance.
int list_reads(hb_ctx* ctx, hb_ctx::Lane* L, const HostBatch& hbt, GatherSizes& gs) {
    const hb_read_store* st = ctx->store;
    if (L->stamp.size() != st->n_reads) { L->stamp.assign(st->n_reads, 0); L->stamp_gen = 0; }
    if (++L->stamp_gen == 0) { std::fill(L->stamp.begin(), L->stamp.end(), 0u); L->stamp_gen = 1; }
    const uint32_t gen = L->stamp_gen;
    PinVec<ReadCopy>& list = L->read_list;
    list.clear();
    if (!list.reserve(std::min<size_t>(hbt.tgt.size() + hbt.ovl.size(), st->n_reads)))
        return fail(ctx, HB_ERR_CAPACITY, "out of pinned host memory (read list)");
    uint64_t dw = 0, dq = 0;
    auto add = [&](uint32_t r) {
        if (L->stamp[r] == gen) return;
        L->stamp[r] = gen;
        const uint32_t len = st->len[r];
        list.p[list.n++] = ReadCopy{st->word_off[r], st->qual_off[r], dw, dq, r, len};
        dw += ((uint64_t)len + 63) / 64 * 2;
        dq += ((uint64_t)len + 15) / 16 * 16;
    };
    for (const DevTarget& t : hbt.tgt) add(t.rid);
    for (const DevOverlap& o : hbt.ovl) add(o.qid);
    gs = GatherSizes{st->n_reads, (uint32_t)list.size(), dw, dq};
    return HB_OK;
}

// The front half of a launch, shared by run_batch and hb_features_batch: carve the batch region for the staged batch, copy it in,
// gather its reads from a host store, and run windowing, the pileup and the per-window lists until the row arena holds every row
// (it is regrown on overflow).  On return `b` views the lane's regions, h.cnt / h.nsup hold the counts of the last attempt,
// ev[0] / ev[2] bracket its feature kernels (the gather included), *total_rows is the rows of all windows, and gs / g describe the
// gather (gs.n_reads == 0 without a host store).
int run_front(hb_ctx* ctx, hb_ctx::Lane* L, const HostBatch& hbt, BatchView& b, Readback& h, uint64_t* launches, uint64_t* total_rows,
              GatherSizes& gs, ReadsInArgs& g, hb_stats& S, double& t_wait, double& t_mark) {
    const uint32_t W = ctx->opt.window_size;
    const size_t nt = hbt.tgt.size(), nw = hbt.win.size();
    const size_t cig_bytes = hbt.cig.size();
    const uint64_t op_slots = hbt.op_cap + hbt.dev_op_cap, raw_slots = hbt.raw_cap;
    if (op_slots >= 0xffffffffull) return fail(ctx, HB_ERR_CAPACITY, "batch too large: more than 2^32 CIGAR ops (lower launch_targets)");
    gs = GatherSizes{};
    g = ReadsInArgs{};
    if (ctx->store) {
        const int rc = list_reads(ctx, L, hbt, gs);
        if (rc) return rc;
        g.src_words = ctx->store_words;
        g.src_qual = ctx->store_qual;
    }
    b = make_view(ctx, hbt);
    CK(L->d_batch.grow(carve_batch(b, cig_bytes, op_slots, raw_slots, gs, g, nullptr)));
    carve_batch(b, cig_bytes, op_slots, raw_slots, gs, g, L->d_batch.as<uint8_t>());
    // ---- H2D straight from the pinned staging arrays of the batch
    const size_t sz[5] = {vbytes(hbt.tgt), vbytes(hbt.win), vbytes(hbt.ovl), vbytes(hbt.ow), hbt.cig.size()};
    const void* src[5] = {hbt.tgt.data(), hbt.win.data(), hbt.ovl.data(), hbt.ow.data(), hbt.cig.data()};
    void* dst[5] = {(void*)b.tgt, (void*)b.win, (void*)b.ovl, b.ow_mut, (void*)b.cig};
    for (int i = 0; i < 5; i++)
        if (sz[i]) CK(cudaMemcpyAsync(dst[i], src[i], sz[i], cudaMemcpyHostToDevice, L->stream));
    S.h2d_bytes += sz[0] + sz[1] + sz[2] + sz[3] + sz[4];

    // a lane's first launch starts with 1.5 W rows per window (HERRO_B200_ARENA_ROWS overrides); later ones keep their arena
    const uint64_t per_win = ctx->arena_rows_per_win ? ctx->arena_rows_per_win : (uint64_t)W + W / 2;
    int rc = set_rows(ctx, L, b, L->rows_cap ? L->rows_cap : (uint64_t)nw * per_win + 64);
    if (rc) return rc;
    CK(L->pin_small.grow(carve_readback(h, nt, nw, nullptr)));
    carve_readback(h, nt, nw, L->pin_small.as<uint8_t>());
    PHASE(0);
    L->kt.on = ctx->time_kernels.load(std::memory_order_relaxed);
    L->kt.st = L->stream;
    for (int attempt = 0;; attempt++) {
        if (attempt) L->kt.discard();
        rc = zero_scratch(ctx, L, b);
        if (rc) return rc;
        CK(cudaEventRecord(L->ev[0], L->stream));
        if (gs.n_reads && attempt == 0) {  // a regrown row arena leaves the batch region, and the gathered reads, as they are
            CK(cudaMemcpyAsync((void*)g.list, L->read_list.data(), vbytes(L->read_list), cudaMemcpyHostToDevice, L->stream));
            *launches += launch_reads_in(g, L->stream, L->kt);
            S.h2d_bytes += vbytes(L->read_list) + gs.words * 8 + gs.qual;
        }
        *launches += launch_features_a(b, L->stream, L->kt);
        CK(cudaEventRecord(L->ev[1], L->stream));
        *launches += launch_pileup(b, L->stream, L->kt, ctx->pileup_v1);
        CK(cudaEventRecord(L->ev[2], L->stream));
        *launches += launch_features_c1(b, L->stream, L->kt);  // ref_lmax + scan; the work list needs its buffers first
        CK(cudaMemcpyAsync(h.cnt, b.counters, CNT_N * 4, cudaMemcpyDeviceToHost, L->stream));
        CK(cudaMemcpyAsync(h.nsup, b.w_nsup, nw * 4, cudaMemcpyDeviceToHost, L->stream));  // the forward passes end at window boundaries
        PHASE(1);
        SYNC_TIMED();
        PHASE(2);
        *total_rows = (uint64_t)h.cnt[CNT_TOTAL_ROWS] | ((uint64_t)h.cnt[CNT_TOTAL_ROWS + 1] << 32);
        if (!h.cnt[CNT_OVERFLOW]) break;
        if (attempt >= 2) return fail(ctx, HB_ERR_CAPACITY, "row arena overflow persisted after regrowth");
        rc = set_rows(ctx, L, b, *total_rows + *total_rows / 8 + 4096);
        if (rc) return rc;
    }
    return HB_OK;
}

int run_batch(hb_ctx* ctx, hb_ctx::Lane* L, HostBatch& hbt) {
    if (hbt.tgt.empty()) return HB_OK;
    const double t_begin = now_ms();
    double t_wait = 0, t_mark = t_begin;
    hb_stats S{};  // merged into ctx->stats under the lock at the end
    std::vector<Result> out_results;
    const uint32_t W = ctx->opt.window_size;
    const size_t nt = hbt.tgt.size(), nw = hbt.win.size();
    // the regions may move below: the view kept from the lane's previous launch would point into freed memory
    L->last.valid = false;
    const size_t cig_bytes = hbt.cig.size();
    const uint64_t op_slots = hbt.op_cap + hbt.dev_op_cap, raw_slots = hbt.raw_cap;
    BatchView b;
    Readback h;
    uint64_t launches = 0;
    uint64_t total_rows = 0;
    GatherSizes gs;
    ReadsInArgs g;
    int rc = run_front(ctx, L, hbt, b, h, &launches, &total_rows, gs, g, S, t_wait, t_mark);
    if (rc) return rc;
    const uint64_t n_sup = (uint64_t)h.cnt[CNT_NSUP] | ((uint64_t)h.cnt[CNT_NSUP + 1] << 32);
    const uint32_t max_nsup = nw ? *std::max_element(h.nsup, h.nsup + nw) : 0;
    FwdBufs f;
    CK(L->d_fwd.grow(carve_fwd(ctx, b, f, n_sup, max_nsup, nullptr)));
    carve_fwd(ctx, b, f, n_sup, max_nsup, L->d_fwd.as<uint8_t>());
    CK(cudaEventRecord(L->ev[3], L->stream));
    rc = launch_tail(ctx, L, b, f, h.nsup, nw, &launches);
    if (rc) return rc;

    // ---- D2H: per-window metadata, then exactly the emitted bytes
    CK(cudaMemcpyAsync(h.cnt, b.counters, CNT_N * 4, cudaMemcpyDeviceToHost, L->stream));
    CK(cudaMemcpyAsync(h.outlen, b.w_outlen, nw * 4, cudaMemcpyDeviceToHost, L->stream));
    CK(cudaMemcpyAsync(h.nsel, b.w_nsel, nw * 4, cudaMemcpyDeviceToHost, L->stream));
    CK(cudaMemcpyAsync(h.L, b.w_L, nw * 4, cudaMemcpyDeviceToHost, L->stream));
    CK(cudaMemcpyAsync(h.terr, b.tgt_err, nt * 4, cudaMemcpyDeviceToHost, L->stream));
    CK(cudaMemcpyAsync(h.sel, b.sel_ow, nw * TOP_K * 4, cudaMemcpyDeviceToHost, L->stream));
    // the emitted bytes of all windows are contiguous from offset 0 and number at most one per matrix row, so the
    // row count (known since the first wait) bounds the copy: no second round trip for the exact size
    CK(L->pin_out.grow(total_rows + 16));
    if (total_rows) CK(cudaMemcpyAsync(L->pin_out.p, b.out_bytes, total_rows, cudaMemcpyDeviceToHost, L->stream));
    PHASE(3);
    SYNC_TIMED();
    PHASE(4);
    const uint64_t total_out = (uint64_t)h.cnt[CNT_TOTAL_OUT] | ((uint64_t)h.cnt[CNT_TOTAL_OUT + 1] << 32);
    if (total_out > total_rows) return fail(ctx, HB_ERR_CAPACITY, "consensus emitted more bytes than matrix rows");
    S.d2h_bytes += CNT_N * 4 + nw * 16 + nt * 4 + nw * TOP_K * 4 + total_rows;

    // ---- timing
    float ms;
    cudaEventElapsedTime(&ms, L->ev[0], L->ev[2]); S.ms_features += ms;
    cudaEventElapsedTime(&ms, L->ev[3], L->ev[4]); S.ms_forward += ms;
    cudaEventElapsedTime(&ms, L->ev[4], L->ev[5]); S.ms_consensus += ms;
    L->kt.collect(S.ms_kernel, S.n_kernel);
    L->kt.on = false;
    add_forward_flops(ctx, S, n_sup, h.nsup, nw);

    // ---- per-read reassembly (src/consensus.rs:90-111,222-226)
    const uint8_t* outb = L->pin_out.as<uint8_t>();
    uint64_t o = 0, corrected = 0, algo = 0;
    for (size_t t = 0; t < nt; t++) {
        const DevTarget& tg = hbt.tgt[t];
        Result r;
        r.rid = tg.rid;
        r.status = HB_OK;
        if (h.terr[t] & TERR_BAD_INPUT) {
            r.status = HB_ERR_INPUT;
            r.msg = "input the reference would panic on (malformed CIGAR / window descriptor / query coordinates)";
        } else if (h.terr[t] & TERR_TOO_MANY_COLS) {
            r.status = HB_ERR_CAPACITY;
            r.msg = "more than " + std::to_string(MAX_COLS_HARD) + " overlap-windows in one window";
        }
        o += append_segments(h.nsel + tg.win_begin, h.outlen + tg.win_begin, tg.win_end - tg.win_begin, outb + o, r.seq, r.seg_len);
        for (uint32_t w = tg.win_begin; w < tg.win_end; w++) {
            // algorithmic bytes of the pileup build for this window (SURVEY.md §8d closed form over the
            // 31 columns the kernel consumes)
            const DevWin& dw = hbt.win[w];
            uint64_t cb = 0;
            for (uint32_t c = 0; c < h.nsel[w]; c++) {
                const DevOW& ow = hbt.ow[h.sel[(size_t)w * TOP_K + c]];
                const DevOverlap& ov = hbt.ovl[ow.ovl];
                if (ov.raw_base == RAW_NONE) cb += ow.cei - ow.csi;
                else cb += (uint64_t)ov.cig_len * W / std::max<uint32_t>(ov.tend - ov.tstart, W);  // device-windowed: its share of the CIGAR
            }
            algo += (uint64_t)(h.nsel[w] + 1) * ((dw.len + 3) / 4 + dw.len) + cb + 2ull * R_COLS * h.L[w];
        }
        if (r.status != HB_OK) { r.seg_len.clear(); r.seq.clear(); }
        corrected += r.seq.size();
        out_results.push_back(std::move(r));
    }
    PHASE(5);
    S.targets += nt;
    S.windows += nw;
    S.overlap_windows += hbt.ow.size();
    S.rows += total_rows;
    S.supported += n_sup;
    S.corrected_bases += corrected;
    S.kernel_launches += launches;
    S.device_launches += 1;
    S.pileup_algo_bytes += algo;

    // ---- publish: results, counters and the metadata for the debug taps / replay
    LastLaunch ll;
    ll.valid = true;
    ll.win.assign(hbt.win.begin(), hbt.win.end());
    ll.w_L.assign(h.L, h.L + nw);
    ll.w_nsel.assign(h.nsel, h.nsel + nw);
    ll.w_nsup.assign(h.nsup, h.nsup + nw);
    ll.w_rowbase.resize(nw);
    ll.w_supbase.resize(nw);
    uint64_t rb = 0, sb = 0;
    for (size_t w = 0; w < nw; w++) {
        ll.w_rowbase[w] = rb; rb += h.L[w];
        ll.w_supbase[w] = sb; sb += h.nsup[w];
        if (ctx->opt.flags & HB_FLAG_KEEP_DEBUG) ll.index[((uint64_t)hbt.win[w].rid << 32) | hbt.win[w].wid] = (uint32_t)w;
    }
    if (ctx->opt.flags & HB_FLAG_KEEP_DEBUG) {
        ll.ow_qid.resize(hbt.ow.size());
        for (size_t i = 0; i < hbt.ow.size(); i++) ll.ow_qid[i] = hbt.ovl[hbt.ow[i].ovl].qid;
    }
    ll.n_sup = n_sup;
    ll.total_rows = total_rows;
    ll.cig_bytes = cig_bytes;
    ll.op_slots = op_slots;
    ll.raw_slots = raw_slots;
    ll.gs = gs;
    ll.view = b;
    ll.fwd = f;
    ll.gather = g;
    S.ms_worker_busy = now_ms() - t_begin;
    S.ms_worker_gpu_wait = t_wait;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        hb_stats& T = ctx->stats;
        T.ms_worker_busy += S.ms_worker_busy; T.ms_worker_gpu_wait += S.ms_worker_gpu_wait;
        T.last_launch_targets = nt; T.last_launch_windows = nw; T.last_launch_bases = corrected;
        T.targets += S.targets; T.windows += S.windows; T.overlap_windows += S.overlap_windows; T.rows += S.rows;
        T.supported += S.supported; T.corrected_bases += S.corrected_bases; T.h2d_bytes += S.h2d_bytes;
        T.d2h_bytes += S.d2h_bytes; T.kernel_launches += S.kernel_launches; T.device_launches += S.device_launches;
        T.pileup_algo_bytes += S.pileup_algo_bytes; T.gemm_flops += S.gemm_flops; T.forward_flops += S.forward_flops;
        T.ms_features += S.ms_features; T.ms_forward += S.ms_forward; T.ms_consensus += S.ms_consensus;
        for (int i = 0; i < HB_NUM_KERNEL_CLASSES; i++) { T.ms_kernel[i] += S.ms_kernel[i]; T.n_kernel[i] += S.n_kernel[i]; T.class_flops[i] += S.class_flops[i]; }
        S.ms_worker_phase[6] = now_ms() - t_mark;
        for (int i = 0; i < 8; i++) T.ms_worker_phase[i] += S.ms_worker_phase[i];
        for (auto& r : out_results) ctx->results.push_back(std::move(r));
        L->last = std::move(ll);
        ctx->last_lane = (int)(L - ctx->lanes);
    }
    return HB_OK;
}

// Hand a staged batch to the launch worker (lock held); `b` is left empty (no capacity).
// Back-pressure: at most 2 batches wait in the queue.
void enqueue_batch(hb_ctx* ctx, std::unique_lock<std::mutex>& lk, HostBatch& b, uint32_t full_targets = 0) {
    // full_targets != 0: several threads submit, and a steady-state hand-over of one of them holds up to that many targets
    if (b.tgt.empty()) return;
    // capacity hint for staging batches: the largest arrays handed over so far plus a margin, so that pinned memory is
    // allocated once per batch object and then recycled.  (No extrapolation from partial batches: a two-target
    // remainder scaled to a full launch once produced hints several times too large, and every pooled batch was then
    // re-pinned inside the next run.)
    const bool first = ctx->cap_hint[0] == 0;
    {
        size_t* h = ctx->cap_hint;
        const size_t cur[5] = {b.tgt.size(), b.win.size(), b.ovl.size(), b.ow.size(), b.cig.size()};
        // Slow start and flush remainders are smaller than a steady-state batch: scale such a batch (at least 32 targets, a fair
        // sample of the per-target sizes) up to the full hand-over size (at most 1 024 targets, at most 16x), so that the pool is
        // pinned once, at its final size, during warm-up.  (A rank of a strong-scaling job only ever hands over remainders whose
        // size depends on how its threads happened to share a step; the largest one seen so far + 25 % was exceeded inside the
        // timed region on 2 of 8 ranks: every pooled batch re-pinned, 51 cudaHostAlloc calls, 1 s.)  Never with a single
        // submitting thread: tests hand over everything in one launch.
        const double scale = (full_targets && cur[0] >= 32 && cur[0] < full_targets) ? std::min(16.0, (double)full_targets / (double)cur[0]) : 1.0;
        for (int i = 0; i < 5; i++) {
            const size_t want = (size_t)((double)cur[i] * scale);
            if (want > h[i]) h[i] = want + want / 4 + 64;
        }
    }
    if (ctx->queue.size() >= 2) {
        const auto t0 = std::chrono::steady_clock::now();
        ctx->cv_idle.wait(lk, [&] { return ctx->queue.size() < 2; });
        g_submit_wait_ns.fetch_add((uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count());
    }
    ctx->queue.push_back(std::move(b));
    b = HostBatch(ctx->device);
    ctx->cv_work.notify_one();
    if (first) {
        // The first hand-over fixes the batch geometry: create the rest of the pool now (lanes in flight + queue + one per
        // submitting thread), so that no staging batch is ever pinned in the steady state whatever the timing of the lanes.
        const uint32_t want = (uint32_t)ctx->n_lanes + 2u + std::max<uint32_t>(ctx->n_slots.load(), 4u);
        size_t h[5];
        for (int i = 0; i < 5; i++) h[i] = ctx->cap_hint[i];
        const uint32_t have = ctx->batches_alive;
        if (want > have) {
            ctx->batches_alive = want;
            lk.unlock();
            std::vector<HostBatch> fresh;
            for (uint32_t i = have; i < want; i++) {
                fresh.emplace_back(ctx->device);
                HostBatch& nb = fresh.back();
                nb.tgt.reserve(h[0]); nb.win.reserve(h[1]); nb.ovl.reserve(h[2]); nb.ow.reserve(h[3]); nb.cig.reserve(h[4]);
            }
            lk.lock();
            for (auto& nb : fresh) ctx->pool.push_back(std::move(nb));
        }
    }
}

// A staging batch with capacity: recycled from the pool, else allocated once at the largest size seen so far
// (pinned allocations are slow and serialise with the worker's CUDA calls, so growth in small steps is avoided).
void acquire_batch(hb_ctx* ctx, HostBatch& b) {
    std::unique_lock<std::mutex> lk(ctx->mu);
    size_t h[5];
    for (int i = 0; i < 5; i++) h[i] = ctx->cap_hint[i];
    if (!ctx->pool.empty()) { b = std::move(ctx->pool.back()); ctx->pool.pop_back(); }
    else { b = HostBatch(ctx->device); ctx->batches_alive++; }
    lk.unlock();
    if (h[0]) { b.tgt.reserve(h[0]); b.win.reserve(h[1]); b.ovl.reserve(h[2]); b.ow.reserve(h[3]); b.cig.reserve(h[4]); }
}

hb_ctx::ThreadSlot* my_slot(hb_ctx* ctx) {
    thread_local hb_ctx* tl_ctx = nullptr;
    thread_local hb_ctx::ThreadSlot* tl_slot = nullptr;
    thread_local uint64_t tl_gen = 0;
    if (tl_ctx == ctx && tl_slot && tl_gen == ctx->generation) return tl_slot;
    std::lock_guard<std::mutex> lk(ctx->mu);
    const auto me = std::this_thread::get_id();
    for (auto& sl : ctx->slots)
        if (sl->owner == me) { tl_ctx = ctx; tl_slot = sl.get(); tl_gen = ctx->generation; return tl_slot; }
    ctx->slots.emplace_back(new hb_ctx::ThreadSlot{me, HostBatch(ctx->device), 0});
    ctx->n_slots.store((uint32_t)ctx->slots.size());
    tl_ctx = ctx; tl_slot = ctx->slots.back().get(); tl_gen = ctx->generation;
    return tl_slot;
}

// Record the capacities this lane ended up with; other lanes grow to them while idle (see hb_ctx::LaneSizes).  Lock held.
void publish_lane_sizes(hb_ctx* ctx, hb_ctx::Lane* L) {
    bool grew = false, below = false;
    hb_ctx::LaneSizes& T = ctx->lane_sizes;
    auto track = [&](size_t& t, size_t have) {
        if (have > t) { t = have; grew = true; }
        below = below || have < t;
    };
    track(T.batch, L->d_batch.cap);
    track(T.rows, L->d_rows.cap);
    track(T.fwd, L->d_fwd.cap);
    track(T.pin_small, L->pin_small.cap);
    track(T.pin_out, L->pin_out.cap);
    track(T.rows_cap, L->rows_cap);
    if (grew) ctx->lane_sizes_version++;
    if (!below) L->seen_sizes = ctx->lane_sizes_version;  // else: this lane catches up when it is next idle
}

// Grow an idle lane's regions to the recorded sizes (no lock held; only this lane's worker touches its regions).
void presize_lane(hb_ctx* ctx, hb_ctx::Lane* L, const hb_ctx::LaneSizes& T) {
    const bool ok = L->d_batch.grow(T.batch, false, true) == cudaSuccess && L->d_rows.grow(T.rows, false, true) == cudaSuccess &&
                    L->d_fwd.grow(T.fwd, false, true) == cudaSuccess && L->pin_small.grow(T.pin_small, false) == cudaSuccess &&
                    L->pin_out.grow(T.pin_out, false) == cudaSuccess;
    if (ok && T.rows_cap > L->rows_cap) L->rows_cap = T.rows_cap;  // T.rows holds a row arena of T.rows_cap rows
    cudaStreamSynchronize(L->stream);
    LastLaunch& ll = L->last;
    if (ll.valid) {  // the regions moved with their contents: carving the kept view's counts again gives the same offsets
        carve_batch(ll.view, ll.cig_bytes, ll.op_slots, ll.raw_slots, ll.gs, ll.gather, L->d_batch.as<uint8_t>());
        carve_rows(ll.view, L->d_rows.as<uint8_t>());
        const uint32_t max_nsup = ll.w_nsup.empty() ? 0 : *std::max_element(ll.w_nsup.begin(), ll.w_nsup.end());
        carve_fwd(ctx, ll.view, ll.fwd, ll.n_sup, max_nsup, L->d_fwd.as<uint8_t>());
    }
}


void worker_main(hb_ctx* ctx, int lane) {
    cudaSetDevice(ctx->device);
    if (ctx->have_node_cpus) pthread_setaffinity_np(pthread_self(), sizeof(cpu_set_t), &ctx->node_cpus);
    hb_ctx::Lane* L = &ctx->lanes[lane];
    std::string my_err;
    t_err_sink = &my_err;
    std::unique_lock<std::mutex> lk(ctx->mu);
    for (;;) {
        ctx->cv_work.wait(lk, [&] { return ctx->stop || !ctx->queue.empty() || L->seen_sizes != ctx->lane_sizes_version; });
        if (ctx->queue.empty()) {
            if (ctx->stop) break;  // stop requested and nothing left
            // idle and another lane has grown: pre-size this lane now rather than inside its next launch
            const hb_ctx::LaneSizes T = ctx->lane_sizes;
            const uint64_t ver = ctx->lane_sizes_version;
            ctx->busy++;  // hb_flush / replay must not run while buffers move
            lk.unlock();
            presize_lane(ctx, L, T);
            lk.lock();
            L->seen_sizes = ver;
            ctx->busy--;
            ctx->cv_idle.notify_all();
            continue;
        }
        HostBatch hbt = std::move(ctx->queue.front());
        ctx->queue.pop_front();
        ctx->busy++;
        ctx->cv_idle.notify_all();
        lk.unlock();
        const int rc = run_batch(ctx, L, hbt);
        lk.lock();
        if (rc != HB_OK) {
            if (ctx->worker_rc == HB_OK) { ctx->worker_rc = rc; ctx->worker_err = my_err; }
            for (const auto& t : hbt.tgt) ctx->results.push_back(Result{t.rid, rc, {}, {}, "launch failed: " + my_err});
        } else {
            const uint64_t before = ctx->lane_sizes_version;
            publish_lane_sizes(ctx, L);
            if (ctx->lane_sizes_version != before) ctx->cv_work.notify_all();
        }
        hbt.clear();
        ctx->pool.push_back(std::move(hbt));
        ctx->busy--;
        ctx->cv_idle.notify_all();
    }
}

// Validation and the per-window bucketing of a target run on the calling (feature) thread without the
// context lock; only the final copy into the shared staging batch is serialised.
struct PreparedTarget {
    uint32_t rid, n_windows, len;
    std::vector<uint32_t> win_begin;  // [n_windows+1] CSR of the bucketed overlap-windows
    std::vector<DevOW> ow;            // bucketed by window, push order kept; ovl/win indices target-local
    uint64_t cig_bytes = 0;
    bool raw = false;                 // device windowing: `ow` is only the (overlap, window) skeleton
    std::vector<uint32_t> aln_now;    // raw: overlap-windows per alignment (0: the alignment contributes nothing, its CIGAR is not shipped)
};

// Which windows an alignment contributes to — the coordinate-only part of windowing::extract_windows
// (src/windowing.rs:53-125,260-272; SURVEY.md App. G steps 1, 2 and 6).  Emitted windows are the contiguous range [wa, we).
// Returns 0, or -1 where the reference would panic (inverted coordinates, a window index past the target's last window,
// the trailing-window unwrap of a None start state).
int skeleton_for_alignment(const hb_overlap& o, uint32_t W, uint32_t n_windows, uint32_t& wa, uint32_t& we) {
    wa = we = 0;
    if (o.tend < o.tstart || o.qend < o.qstart) return -1;
    if (o.tend - o.tstart < W || o.qend - o.qstart < W) return 0;          // :53-57
    const uint32_t edge = (uint32_t)(0.1f * (float)W);                      // :65
    if (o.tlen < edge) return -1;
    const uint32_t tail_thresh = o.tlen - edge;
    const uint32_t first_w = o.tstart < edge ? 0 : (o.tstart + W - 1) / W;  // :75-79
    const uint32_t last_w = o.tend > tail_thresh ? (o.tend - 1) / W + 1 : o.tend / W;  // :81-85
    if (last_w <= first_w) return 0;                                       // :106
    const bool open0 = (o.tstart % W == 0) || (o.tstart < edge);            // :120-125
    const uint32_t w_cur = o.tstart / W, w_new = o.tend / W;
    const uint32_t a = open0 ? w_cur : w_cur + 1;  // a window is emitted at every boundary crossed once a start state exists
    uint32_t e = w_new;
    if (o.tend > tail_thresh && o.tend % W != 0) {  // trailing partial window
        if (!open0 && w_new == w_cur) return -1;    // the reference unwraps a None start state here
        e = w_new + 1;
    }
    if (e <= a) return 0;
    if (e > n_windows) return -1;
    wa = a; we = e;
    return 0;
}

int prepare_target(hb_ctx* ctx, uint32_t rid, uint32_t n_windows, const hb_overlap* ovl, uint32_t n_ovl,
                   const hb_overlap_window* ow, uint32_t n_ow, PreparedTarget& P) {
    if (!ctx->have_reads) return fail(ctx, HB_ERR_STATE, "hb_upload_reads must be called before submitting targets");
    if (rid >= ctx->n_reads) return fail(ctx, HB_ERR_ARG, "rid out of range");
    const uint32_t W = ctx->opt.window_size;
    const uint32_t len = ctx->read_len[rid];
    if (n_windows != (len + W - 1) / W) return fail(ctx, HB_ERR_ARG, "n_windows != ceil(read_len / window_size)");
    if ((n_ovl && !ovl) || (n_ow && !ow)) return fail(ctx, HB_ERR_ARG, "null array");
    uint64_t cb = 0;
    for (uint32_t i = 0; i < n_ovl; i++) {
        if (ovl[i].tid != rid) return fail(ctx, HB_ERR_ARG, "overlap.tid != rid (alignments must be grouped by target)");
        if (ovl[i].qid >= ctx->n_reads) return fail(ctx, HB_ERR_ARG, "overlap.qid out of range");
        if (!ovl[i].cigar && ovl[i].cigar_len) return fail(ctx, HB_ERR_ARG, "null cigar");
        if (ovl[i].strand > 1) return fail(ctx, HB_ERR_ARG, "strand must be 0 or 1");
        cb += ovl[i].cigar_len;
    }
    P.rid = rid; P.n_windows = n_windows; P.len = len; P.cig_bytes = cb;
    P.win_begin.assign(n_windows + 1, 0);
    for (uint32_t i = 0; i < n_ow; i++) {
        if (ow[i].overlap_idx >= n_ovl || ow[i].window_idx >= n_windows) return fail(ctx, HB_ERR_ARG, "overlap_window index out of range");
        if (ow[i].cigar_end_idx < ow[i].cigar_start_idx || ow[i].cigar_end_idx > ovl[ow[i].overlap_idx].cigar_len)
            return fail(ctx, HB_ERR_ARG, "overlap_window cigar range out of bounds");
        P.win_begin[ow[i].window_idx + 1]++;
    }
    for (uint32_t w = 0; w < n_windows; w++) P.win_begin[w + 1] += P.win_begin[w];
    // bucket by window, keeping push order (= alignment order) inside each
    P.ow.resize(n_ow);
    thread_local std::vector<uint32_t> fill;  // scratch reused across calls: no allocation per target
    fill.assign(P.win_begin.begin(), P.win_begin.end() - 1);
    for (uint32_t i = 0; i < n_ow; i++) {
        const hb_overlap_window& s = ow[i];
        P.ow[fill[s.window_idx]++] = DevOW{s.overlap_idx, s.window_idx, s.tstart, s.qstart, s.qend, s.cigar_start_idx,
                                           s.cigar_start_offset, s.cigar_end_idx, s.cigar_end_offset, 0};
    }
    return HB_OK;
}

int append_target(hb_ctx* ctx, HostBatch& hbt, const PreparedTarget& P, const hb_overlap* ovl, uint32_t n_ovl) {
    const uint32_t W = ctx->opt.window_size;
    const uint32_t t_idx = (uint32_t)hbt.tgt.size();
    const uint32_t ovl_base = (uint32_t)hbt.ovl.size(), win_base = (uint32_t)hbt.win.size(), ow_base = (uint32_t)hbt.ow.size();
    const uint32_t n_ow = (uint32_t)P.ow.size();
    if (!hbt.ovl.reserve(ovl_base + n_ovl) || !hbt.cig.reserve(hbt.cig.size() + P.cig_bytes) || !hbt.win.reserve(win_base + P.n_windows) ||
        !hbt.ow.resize(ow_base + n_ow) || !hbt.tgt.reserve(t_idx + 1))
        return fail(ctx, HB_ERR_CAPACITY, "out of pinned host memory");
    for (uint32_t i = 0; i < n_ovl; i++) {
        DevOverlap d{ovl[i].qid, ovl[i].qstart, ovl[i].qend, ovl[i].strand, (uint64_t)hbt.cig.size(), ovl[i].cigar_len, t_idx,
                     ovl[i].tstart, ovl[i].tend, RAW_NONE, 0};
        if (P.raw) {
            if (P.aln_now[i] == 0) {
                d.cig_len = 0;  // contributes to no window: its CIGAR stays on the host
            } else {
                d.raw_base = (uint32_t)hbt.raw_cap;
                hbt.raw_cap += ovl[i].cigar_len / 2 + 1;
                hbt.dev_op_cap += ovl[i].cigar_len / 2 + 1 + P.aln_now[i];  // every op once + one shared op per boundary
                hbt.n_raw++;
                hbt.cig.append(ovl[i].cigar, ovl[i].cigar_len);
            }
        } else {
            hbt.cig.append(ovl[i].cigar, ovl[i].cigar_len);
        }
        hbt.ovl.push_back(d);
    }
    for (uint32_t w = 0; w < P.n_windows; w++) {
        DevWin d{};
        d.tgt = t_idx; d.rid = P.rid; d.wid = w; d.tstart = w * W;
        d.len = (w == P.n_windows - 1) ? P.len - w * W : W;
        d.ow_begin = ow_base + P.win_begin[w];
        d.ow_end = ow_base + P.win_begin[w + 1];
        hbt.win.push_back(d);
    }
    uint64_t opc = hbt.op_cap;
    for (uint32_t i = 0; i < n_ow; i++) {
        DevOW d = P.ow[i];
        d.ovl += ovl_base;
        d.win += win_base;
        if (P.raw) {
            d.op_base = 0;  // assigned on the device
        } else {
            d.op_base = (uint32_t)opc;
            opc += (d.cei - d.csi) / 2 + 1;
        }
        hbt.ow[ow_base + i] = d;
    }
    hbt.op_cap = opc;
    hbt.tgt.push_back(DevTarget{P.rid, win_base, win_base + P.n_windows, ovl_base, ovl_base + n_ovl});
    return HB_OK;
}

// Stage one prepared target in the calling thread's batch and hand the batch over when it is full.
int stage_target(hb_ctx* ctx, const PreparedTarget& P, const hb_overlap* ovl, uint32_t n_ovl) {
    hb_ctx::ThreadSlot* slot = my_slot(ctx);
    if (slot->batch.tgt.cap == 0) acquire_batch(ctx, slot->batch);
    std::string local_err;
    t_err_sink = &local_err;
    const int rc = append_target(ctx, slot->batch, P, ovl, n_ovl);
    t_err_sink = nullptr;
    if (rc) { std::lock_guard<std::mutex> lk(ctx->mu); ctx->err = local_err; return rc; }
    // `launch_targets` is shared by the submitting threads: each stages launch_targets / n_threads targets per launch,
    // so the targets in flight (and the latency to the first launch) do not grow with the thread count
    const uint32_t lt = ctx->opt.launch_targets, ns = std::max(1u, ctx->n_slots.load(std::memory_order_relaxed));
    // ... but never less than 256 targets per launch (unless launch_targets itself is smaller): ~1 300 windows is what it takes to
    // fill the 132 SMs of an H100 with the one-CTA-per-window feature kernels and to amortise the ~25 launches of a batch
    uint32_t thr = std::min(lt, std::max(ctx->min_launch, lt / ns));
    // slow start: with several submitting threads, the first hand-overs after a flush are small and grow geometrically (48, 72, 108, ...
    // targets, counted over all threads), so that the GPU has work a few milliseconds after the first submit instead of after a
    // whole launch has been staged, and the threads - which fill their batches at the same rate - do not all hand over at the
    // same moment.  (A single submitting thread keeps exact launch sizes: tests and the isolated launch bench.py times rely on
    // them.)  Matters when a run is short: a rank of an 8-GPU strong-scaling job sees ~100 ms of work.
    const uint32_t full_thr = thr;
    if (ns >= 2) {
        static const uint16_t ramp[5] = {48, 72, 108, 162, 243};
        const uint32_t n = ctx->handed_total.load(std::memory_order_relaxed);
        if (n < 5) thr = std::min<uint32_t>(thr, ramp[n]);
    }
    if (slot->batch.tgt.size() >= thr) {
        std::unique_lock<std::mutex> lk(ctx->mu);
        enqueue_batch(ctx, lk, slot->batch, ns >= 2 ? std::min(full_thr, 1024u) : 0u);
        slot->handed++;
        ctx->handed_total.fetch_add(1, std::memory_order_relaxed);
    }
    return HB_OK;
}

// The target preparation of hb_submit_alignments, shared with hb_features_batch: checks the alignments of target `rid` and lays
// out the target's overlap-windows in P.  HB_ERR_INPUT: coordinates (or, with host windowing, a CIGAR) the reference would panic
// on; any other error is the caller's.
int prepare_alignments(hb_ctx* ctx, uint32_t rid, const hb_overlap* ovl, uint32_t n_ovl, PreparedTarget& P) {
    if (!ctx->have_reads) return fail(ctx, HB_ERR_STATE, "hb_upload_reads must be called before submitting targets");
    if (rid >= ctx->n_reads) return fail(ctx, HB_ERR_ARG, "rid out of range");
    if (n_ovl && !ovl) return fail(ctx, HB_ERR_ARG, "null array");
    const uint32_t W = ctx->opt.window_size;
    const uint32_t n_windows = (ctx->read_len[rid] + W - 1) / W;
    if (ctx->host_windowing) {  // A-B path: extract_windows on the calling thread, then the hb_submit_target route
        thread_local std::vector<hb_overlap_window> ows;
        ows.clear();
        for (uint32_t i = 0; i < n_ovl; i++) {
            if (ovl[i].tid != rid) return fail(ctx, HB_ERR_ARG, "overlap.tid != rid");
            if (host_extract_windows(ovl[i], i, W, n_windows, ows) != 0)
                return fail(ctx, HB_ERR_INPUT, "malformed alignment (CIGAR / coordinates) for target " + std::to_string(rid));
        }
        P.raw = false;
        return prepare_target(ctx, rid, n_windows, ovl, n_ovl, ows.data(), (uint32_t)ows.size(), P);
    }
    // Device windowing (windowing_dev.cu): the host only lays out which (alignment, window) pairs exist — a function of the PAF
    // coordinates — and ships the CIGARs; a CIGAR that is malformed or disagrees with its coordinates fails this target on the
    // device (tgt_err) instead of here.
    thread_local std::vector<uint32_t> first, fill;
    P.raw = true;
    P.rid = rid; P.n_windows = n_windows; P.len = ctx->read_len[rid];
    P.win_begin.assign(n_windows + 1, 0);
    P.aln_now.assign(n_ovl, 0);
    first.assign(n_ovl, 0);
    uint64_t cb = 0;
    for (uint32_t i = 0; i < n_ovl; i++) {
        if (ovl[i].tid != rid) return fail(ctx, HB_ERR_ARG, "overlap.tid != rid (alignments must be grouped by target)");
        if (ovl[i].qid >= ctx->n_reads) return fail(ctx, HB_ERR_ARG, "overlap.qid out of range");
        if (!ovl[i].cigar && ovl[i].cigar_len) return fail(ctx, HB_ERR_ARG, "null cigar");
        if (ovl[i].strand > 1) return fail(ctx, HB_ERR_ARG, "strand must be 0 or 1");
        uint32_t wa, we;
        if (skeleton_for_alignment(ovl[i], W, n_windows, wa, we) != 0)
            return fail(ctx, HB_ERR_INPUT, "malformed alignment (coordinates) for target " + std::to_string(rid));
        first[i] = wa;
        P.aln_now[i] = we - wa;
        if (we > wa) cb += ovl[i].cigar_len;
        for (uint32_t w = wa; w < we; w++) P.win_begin[w + 1]++;
    }
    for (uint32_t w = 0; w < n_windows; w++) P.win_begin[w + 1] += P.win_begin[w];
    P.cig_bytes = cb;
    P.ow.resize(P.win_begin[n_windows]);
    fill.assign(P.win_begin.begin(), P.win_begin.end() - 1);
    for (uint32_t i = 0; i < n_ovl; i++)  // alignment order inside every window = the reference's push order
        for (uint32_t w = first[i]; w < first[i] + P.aln_now[i]; w++) P.ow[fill[w]++] = DevOW{i, w, 0, 0, 0, 0, 0, 0, 0, 0};
    return HB_OK;
}

int no_model_fail(hb_ctx* ctx) {
    std::lock_guard<std::mutex> lk(ctx->mu);
    return fail(ctx, HB_ERR_STATE, "the context was created with HB_FLAG_NO_MODEL: it has no weights to run the forward with");
}

// ---------------------------------------------------------------------------------- hb_forward_batch
// Its input region: the caller's tokens and qualities (host path only: in_bytes is 0 otherwise), the per-window arrays of the
// view and the error word.  Carved alike in pinned and in device memory, so one copy moves all of it.
struct FwdIn {
    uint8_t *tok, *qual;
    uint32_t *L, *nsup, *nsel;
    uint64_t *rowbase, *supbase;
    unsigned long long* bad;
};
size_t carve_fwd_in(FwdIn& a, size_t in_bytes, size_t nb, uint8_t* base) {
    Carve c{base};
    c(a.tok, in_bytes);
    c(a.qual, in_bytes);
    c(a.L, nb);
    c(a.nsup, nb);
    c(a.nsel, nb);
    c(a.rowbase, nb);
    c(a.supbase, nb);
    c(a.bad, 1);
    return c.bytes;
}

// Where a caller's pointer lives: 1 device memory of `device` (or managed), -1 another device's memory, 0 host memory
int pointer_kind(const void* p, int device) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return 0; }
    if (at.type == cudaMemoryTypeManaged) return 1;
    if (at.type != cudaMemoryTypeDevice) return 0;
    return at.device == device ? 1 : -1;
}

// The work of hb_forward_batch, with the lane's lock held and the context's device current
int forward_batch(hb_ctx* ctx, uint32_t B, uint32_t Lmax, const uint8_t* bases, const uint8_t* quals, const int32_t* lens,
                  const int32_t* indices, float* info_out, float* logits_out, uint32_t flags, void* stream) {
    hb_ctx::FwdLane& F = ctx->fwd;
    if (!bases || !quals || !lens || !indices || !info_out || !logits_out) return fail(ctx, HB_ERR_ARG, "null pointer");
    if (B == 0 || Lmax == 0) return fail(ctx, HB_ERR_ARG, "B and Lmax must be positive");
    if (flags & ~HB_FWD_DEVICE_PTRS) return fail(ctx, HB_ERR_ARG, "unknown flags");
    const bool dev = (flags & HB_FWD_DEVICE_PTRS) != 0;
    {
        const void* p[6] = {bases, quals, info_out, logits_out, lens, indices};
        static const char* name[6] = {"bases", "quals", "info_logits", "bases_logits", "lens", "indices"};
        for (int i = 0; i < 6; i++) {
            const int k = pointer_kind(p[i], ctx->device);
            if (dev && i < 4 && k != 1)
                return fail(ctx, HB_ERR_ARG, std::string(name[i]) + " is not memory of device " + std::to_string(ctx->device) +
                                                 " (HB_FWD_DEVICE_PTRS is set)");
            if ((!dev || i >= 4) && k != 0)
                return fail(ctx, HB_ERR_ARG, std::string(name[i]) + " is device memory" + (i < 4 ? " (HB_FWD_DEVICE_PTRS is not set)" : ""));
        }
    }
    uint64_t n = 0;
    uint32_t max_len = 0;
    for (uint32_t b = 0; b < B; b++) {
        if (lens[b] < 0) return fail(ctx, HB_ERR_ARG, "lens[" + std::to_string(b) + "] is negative");
        n += (uint64_t)lens[b];
        max_len = std::max(max_len, (uint32_t)lens[b]);
    }
    if (n == 0) return HB_OK;
    const uint64_t rows = (uint64_t)B * Lmax;
    if (n >= (1ull << 31) || rows >= (1ull << 36)) return fail(ctx, HB_ERR_CAPACITY, "batch too large");
    // ---- scratch (grow-only) and the view
    const size_t in_bytes = dev ? 0 : (size_t)rows * R_COLS;
    FwdIn hp, dp;
    const size_t in_sz = carve_fwd_in(hp, in_bytes, B, nullptr);
    CK(F.pin_in.grow(in_sz + 2 * al256(n * 4)));
    carve_fwd_in(hp, in_bytes, B, F.pin_in.as<uint8_t>());
    uint32_t* h_win = (uint32_t*)(F.pin_in.as<uint8_t>() + in_sz);
    uint32_t* h_row = (uint32_t*)((uint8_t*)h_win + al256(n * 4));
    CK(F.d_in.grow(in_sz));
    carve_fwd_in(dp, in_bytes, B, F.d_in.as<uint8_t>());
    BatchView b{};
    b.n_win = B;
    b.w_L = b.w_reflmax = dp.L;  // every window is Lmax rows long, and so is its batch
    b.w_nsup = dp.nsup;
    b.w_nsel = dp.nsel;          // 0: k_heads writes no consensus byte
    b.w_rowbase = dp.rowbase;
    b.w_supbase = dp.supbase;
    CK(F.d_mat.grow(2 * al256(rows * ROW_BYTES)));
    b.mat_bases = F.d_mat.as<uint8_t>();
    b.mat_quals = b.mat_bases + al256(rows * ROW_BYTES);
    FwdBufs f;
    CK(F.d_fwd.grow(carve_fwd(ctx, b, f, n, max_len, nullptr)));
    carve_fwd(ctx, b, f, n, max_len, F.d_fwd.as<uint8_t>());
    float *h_info = nullptr, *h_logits = nullptr;
    if (!dev) {
        CK(F.pin_out.grow(al256(n * 4) + n * 20));
        h_info = F.pin_out.as<float>();
        h_logits = (float*)(F.pin_out.as<uint8_t>() + al256(n * 4));
    }
    // ---- the per-window arrays and the work list, checking every index
    uint64_t sb = 0;
    for (uint32_t w = 0; w < B; w++) {
        hp.L[w] = Lmax;
        hp.nsup[w] = (uint32_t)lens[w];
        hp.nsel[w] = 0;
        hp.rowbase[w] = (uint64_t)w * Lmax;
        hp.supbase[w] = sb;
        for (uint32_t k = 0; k < (uint32_t)lens[w]; k++) {
            const int32_t r = indices[sb + k];
            if (r < 0 || (uint32_t)r >= Lmax)
                return fail(ctx, HB_ERR_ARG, "indices[" + std::to_string(sb + k) + "] = " + std::to_string(r) + " (window " + std::to_string(w) +
                                                 ") is outside [0, Lmax = " + std::to_string(Lmax) + ")");
            h_win[sb + k] = w;
            h_row[sb + k] = (uint32_t)r;
        }
        sb += (uint32_t)lens[w];
    }
    *hp.bad = ~0ull;
    if (!dev) {
        memcpy(hp.tok, bases, in_bytes);
        memcpy(hp.qual, quals, in_bytes);
    }
    // ---- device work
    KTimer& kt = F.kt;
    kt.discard();
    kt.on = ctx->time_kernels.load(std::memory_order_relaxed);
    kt.st = F.stream;
    if (dev) {
        CK(cudaEventRecord(F.ev[0], (cudaStream_t)stream));
        CK(cudaStreamWaitEvent(F.stream, F.ev[0], 0));
    }
    CK(cudaMemcpyAsync(F.d_in.p, F.pin_in.p, in_sz, cudaMemcpyHostToDevice, F.stream));
    CK(cudaMemcpyAsync(b.fwd_win, h_win, n * 4, cudaMemcpyHostToDevice, F.stream));
    CK(cudaMemcpyAsync(b.fwd_row, h_row, n * 4, cudaMemcpyHostToDevice, F.stream));
    CK(cudaEventRecord(F.ev[1], F.stream));
    kt.begin(K_LISTS);
    launch_batch_in(dev ? bases : dp.tok, dev ? quals : dp.qual, rows, b.mat_bases, b.mat_quals, dp.bad, F.stream);
    kt.end();
    const uint64_t launches = 1 + launch_forward_passes(ctx, b, f, hp.nsup, B, F.stream, kt);
    CK(cudaGetLastError());
    CK(cudaEventRecord(F.ev[2], F.stream));
    CK(cudaMemcpyAsync(hp.bad, dp.bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, F.stream));
    if (!dev) {
        CK(cudaMemcpyAsync(h_info, f.info, n * 4, cudaMemcpyDeviceToHost, F.stream));
        CK(cudaMemcpyAsync(h_logits, f.logits, n * 20, cudaMemcpyDeviceToHost, F.stream));
    }
    CK(cudaStreamSynchronize(F.stream));
    if (*hp.bad != ~0ull) {
        kt.discard();
        const uint64_t e = *hp.bad, per = (uint64_t)Lmax * R_COLS;
        return fail(ctx, HB_ERR_INPUT, "token above 11 at (b, row, col) = (" + std::to_string(e / per) + ", " + std::to_string(e % per / R_COLS) +
                                            ", " + std::to_string(e % R_COLS) + "): the model's embedding has 12 entries");
    }
    if (dev) {
        CK(cudaMemcpyAsync(info_out, f.info, n * 4, cudaMemcpyDeviceToDevice, F.stream));
        CK(cudaMemcpyAsync(logits_out, f.logits, n * 20, cudaMemcpyDeviceToDevice, F.stream));
        CK(cudaStreamSynchronize(F.stream));
    } else {
        memcpy(info_out, h_info, n * 4);
        memcpy(logits_out, h_logits, n * 20);
    }
    // ---- counters
    hb_stats S{};
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, F.ev[1], F.ev[2]));
    kt.collect(S.ms_kernel, S.n_kernel);
    kt.on = false;
    add_forward_flops(ctx, S, n, hp.nsup, B);
    std::lock_guard<std::mutex> lk(ctx->mu);
    hb_stats& T = ctx->stats;
    T.ms_forward += ms;
    T.supported += n;
    T.kernel_launches += launches;
    T.gemm_flops += S.gemm_flops;
    T.forward_flops += S.forward_flops;
    for (int i = 0; i < HB_NUM_KERNEL_CLASSES; i++) { T.ms_kernel[i] += S.ms_kernel[i]; T.n_kernel[i] += S.n_kernel[i]; T.class_flops[i] += S.class_flops[i]; }
    return HB_OK;
}

// ---------------------------------------------------------------------------------- hb_consensus_batch
// Its input region: the caller's tokens and logits (host path only: both byte counts are 0 otherwise), the windows' keys, the
// per-window arrays and the error word.  Carved alike in pinned and in device memory, so one copy moves all of it.
struct ConsIn {
    uint8_t* tok;
    float* logits;
    uint2* keys;
    uint32_t *L, *nsel, *nkeys;
    uint64_t *rowbase, *keybase;
    unsigned long long* bad;
};
size_t carve_cons_in(ConsIn& a, size_t tok_bytes, size_t logit_rows, size_t n_keys, size_t nw, uint8_t* base) {
    Carve c{base};
    c(a.tok, tok_bytes);
    c(a.logits, logit_rows * 5);
    c(a.keys, std::max<size_t>(n_keys, 1));
    c(a.L, nw);
    c(a.nsel, nw);
    c(a.nkeys, nw);
    c(a.rowbase, nw);
    c(a.keybase, nw);
    c(a.bad, 1);
    return c.bytes;
}
// The consensus region: the rows' emit bytes and the pipeline's consensus arrays (k_cons_count, the scan, k_cons_write)
size_t carve_cons_out(BatchView& b, size_t rows, size_t nw, uint8_t* base) {
    Carve c{base};
    c(b.row_emit, std::max<size_t>(rows, 1));
    c(b.out_bytes, std::max<size_t>(rows, 1));
    c(b.w_outlen, nw);
    c(b.w_outoff, nw);
    c(b.counters, CNT_N);
    return c.bytes;
}

// The work of hb_consensus_batch, with the lane's lock held and the context's device current
int consensus_batch(hb_ctx* ctx, uint32_t n_reads, const uint32_t* n_windows, const uint32_t* rows, const uint8_t* n_alns,
                    const uint8_t* bases, const uint32_t* n_sup, const uint32_t* supported, const float* bases_logits, uint8_t* seqs,
                    uint32_t* seg_len, uint32_t* n_segs, uint32_t flags, void* stream) {
    hb_ctx::ConsLane& Cn = ctx->cons;
    if (!n_windows || !rows || !n_alns || !bases || !n_sup || !supported || !bases_logits || !seqs || !seg_len || !n_segs)
        return fail(ctx, HB_ERR_ARG, "null pointer");
    if (flags & ~HB_CONS_DEVICE_PTRS) return fail(ctx, HB_ERR_ARG, "unknown flags");
    const bool dev = (flags & HB_CONS_DEVICE_PTRS) != 0;
    {
        const void* p[10] = {bases, bases_logits, n_windows, rows, n_alns, n_sup, supported, seqs, seg_len, n_segs};
        static const char* name[10] = {"bases", "bases_logits", "n_windows", "rows", "n_alns", "n_sup", "supported", "seqs", "seg_len", "n_segs"};
        for (int i = 0; i < 10; i++) {
            const int k = pointer_kind(p[i], ctx->device);
            if (dev && i < 2 && k != 1)
                return fail(ctx, HB_ERR_ARG, std::string(name[i]) + " is not memory of device " + std::to_string(ctx->device) +
                                                 " (HB_CONS_DEVICE_PTRS is set)");
            if ((!dev || i >= 2) && k != 0)
                return fail(ctx, HB_ERR_ARG, std::string(name[i]) + " is device memory" + (i < 2 ? " (HB_CONS_DEVICE_PTRS is not set)" : ""));
        }
    }
    // ---- sizes and range checks
    uint64_t nw = 0;
    for (uint32_t i = 0; i < n_reads; i++) nw += n_windows[i];
    if (nw >= (1ull << 31)) return fail(ctx, HB_ERR_CAPACITY, "batch too large: 2^31 windows or more");
    uint64_t n_rows = 0, n_pos = 0;
    for (uint64_t w = 0; w < nw; w++) {
        if (n_alns[w] > TOP_K)
            return fail(ctx, HB_ERR_ARG, "n_alns[" + std::to_string(w) + "] = " + std::to_string(n_alns[w]) + " is above " + std::to_string(TOP_K));
        n_rows += rows[w];
        n_pos += n_sup[w];
    }
    for (uint64_t k = 0; k < n_pos; k++)
        if (supported[2 * k] > 0xffffu || supported[2 * k + 1] > 0xffu)
            return fail(ctx, HB_ERR_ARG, "supported[" + std::to_string(k) + "] = (" + std::to_string(supported[2 * k]) + ", " +
                                             std::to_string(supported[2 * k + 1]) + ") is not a (u16 pos, u8 ins) SupportedPos");
    if (n_pos >= (1ull << 32) || n_rows >= (1ull << 40)) return fail(ctx, HB_ERR_CAPACITY, "batch too large");
    if (nw == 0) {
        memset(n_segs, 0, (size_t)n_reads * 4);
        return HB_OK;
    }
    // ---- scratch (grow-only)
    const size_t tok_bytes = dev ? 0 : (size_t)n_rows * R_COLS, logit_rows = dev ? 0 : (size_t)n_pos;
    ConsIn hp, dp;
    const size_t in_sz = carve_cons_in(hp, tok_bytes, logit_rows, n_pos, nw, nullptr);
    CK(Cn.pin_in.grow(in_sz));
    carve_cons_in(hp, tok_bytes, logit_rows, n_pos, nw, Cn.pin_in.as<uint8_t>());
    CK(Cn.d_in.grow(in_sz));
    carve_cons_in(dp, tok_bytes, logit_rows, n_pos, nw, Cn.d_in.as<uint8_t>());
    BatchView b{};
    b.n_win = (uint32_t)nw;
    b.w_L = dp.L;
    b.w_nsel = dp.nsel;
    b.w_rowbase = dp.rowbase;
    CK(Cn.d_out.grow(carve_cons_out(b, n_rows, nw, nullptr)));
    carve_cons_out(b, n_rows, nw, Cn.d_out.as<uint8_t>());
    const size_t out_sz = al256(nw * 4) + n_rows;
    CK(Cn.pin_out.grow(out_sz));
    uint32_t* h_outlen = Cn.pin_out.as<uint32_t>();
    const uint8_t* h_bytes = Cn.pin_out.as<uint8_t>() + al256(nw * 4);
    // ---- the per-window arrays and the keys: (pos << 8 | ins, logit row) sorted by key, the last of equal keys kept (the
    // HashMap collect of src/consensus.rs:115-124).  The features stage emits a window's positions in row order, so its keys are
    // strictly increasing and one pass confirms it; anything else is sorted.
    uint64_t rb = 0, sb = 0, kb = 0;
    for (uint64_t w = 0; w < nw; w++) {
        hp.L[w] = rows[w];
        hp.nsel[w] = n_alns[w];
        hp.rowbase[w] = rb;
        hp.keybase[w] = kb;
        const uint32_t ns = n_sup[w];
        const uint32_t* sp = supported + 2 * sb;
        uint32_t nk = 0;
        if (n_alns[w] >= 2 && ns) {
            auto key = [&](uint32_t j) { return sp[2 * j] << 8 | sp[2 * j + 1]; };
            bool sorted = true;
            for (uint32_t j = 1; j < ns && sorted; j++) sorted = key(j - 1) < key(j);
            if (sorted) {
                for (uint32_t j = 0; j < ns; j++) hp.keys[kb + j] = make_uint2(key(j), (uint32_t)(sb + j));
                nk = ns;
            } else {
                Cn.order.resize(ns);
                for (uint32_t j = 0; j < ns; j++) Cn.order[j] = j;
                std::stable_sort(Cn.order.begin(), Cn.order.end(), [&](uint32_t x, uint32_t y) { return key(x) < key(y); });
                for (uint32_t i = 0; i < ns; i++) {
                    const uint32_t j = Cn.order[i];
                    if (i + 1 < ns && key(Cn.order[i + 1]) == key(j)) continue;  // a later duplicate replaces this one
                    hp.keys[kb + nk++] = make_uint2(key(j), (uint32_t)(sb + j));
                }
            }
        }
        hp.nkeys[w] = nk;
        rb += rows[w];
        sb += ns;
        kb += nk;
    }
    *hp.bad = ~0ull;
    if (!dev) {
        memcpy(hp.tok, bases, tok_bytes);
        memcpy(hp.logits, bases_logits, (size_t)n_pos * 20);
    }
    // ---- device work
    KTimer& kt = Cn.kt;
    kt.discard();
    kt.on = ctx->time_kernels.load(std::memory_order_relaxed);
    kt.st = Cn.stream;
    if (dev) {
        CK(cudaEventRecord(Cn.ev[0], (cudaStream_t)stream));
        CK(cudaStreamWaitEvent(Cn.stream, Cn.ev[0], 0));
    }
    CK(cudaMemcpyAsync(Cn.d_in.p, Cn.pin_in.p, in_sz, cudaMemcpyHostToDevice, Cn.stream));
    CK(cudaEventRecord(Cn.ev[1], Cn.stream));
    const ConsInArgs ca{dev ? bases : dp.tok, dev ? bases_logits : dp.logits, dp.keys, dp.L, dp.nsel, dp.rowbase, dp.keybase, dp.nkeys,
                        b.row_emit, dp.bad};
    kt.begin(K_CONSENSUS);
    launch_cons_in(ca, (uint32_t)nw, Cn.stream);
    kt.end();
    const uint64_t launches = 1 + launch_consensus(b, Cn.stream, kt);
    CK(cudaGetLastError());
    CK(cudaEventRecord(Cn.ev[2], Cn.stream));
    CK(cudaMemcpyAsync(hp.bad, dp.bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, Cn.stream));
    CK(cudaMemcpyAsync(h_outlen, b.w_outlen, nw * 4, cudaMemcpyDeviceToHost, Cn.stream));
    // the emitted bytes number at most one per row: the row count bounds the copy, as in the pipeline
    if (n_rows) CK(cudaMemcpyAsync((void*)h_bytes, b.out_bytes, n_rows, cudaMemcpyDeviceToHost, Cn.stream));
    CK(cudaStreamSynchronize(Cn.stream));
    if (*hp.bad != ~0ull) {
        kt.discard();
        const uint64_t e = *hp.bad, row = e / R_COLS, col = e % R_COLS;
        const uint64_t w = (uint64_t)(std::upper_bound(hp.rowbase, hp.rowbase + nw, row) - hp.rowbase) - 1;
        uint64_t r = 0, w0 = 0;
        while (w0 + n_windows[r] <= w) w0 += n_windows[r++];
        const uint8_t tok = dev ? 0 : hp.tok[e];
        return fail(ctx, HB_ERR_INPUT, "consensus() would panic at (read, window, row, column) = (" + std::to_string(r) + ", " +
                                           std::to_string(w - w0) + ", " + std::to_string(row - hp.rowbase[w]) + ", " + std::to_string(col) +
                                           (dev ? std::string(")") : "), token " + std::to_string(tok)) +
                                           (col == 0 ? ": no BASES_UPPER entry for the target column" : ": no BASES_UPPER_COUNTER entry"));
    }
    // ---- per-read segments, then the caller's outputs
    Cn.seq.clear();
    Cn.seg_len.clear();
    uint64_t o = 0, w0 = 0;
    for (uint32_t i = 0; i < n_reads; i++) {
        const size_t s0 = Cn.seg_len.size();
        o += append_segments(hp.nsel + w0, h_outlen + w0, n_windows[i], h_bytes + o, Cn.seq, Cn.seg_len);
        n_segs[i] = (uint32_t)(Cn.seg_len.size() - s0);
        w0 += n_windows[i];
    }
    if (!Cn.seq.empty()) memcpy(seqs, Cn.seq.data(), Cn.seq.size());
    if (!Cn.seg_len.empty()) memcpy(seg_len, Cn.seg_len.data(), Cn.seg_len.size() * 4);
    // ---- counters
    hb_stats S{};
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, Cn.ev[1], Cn.ev[2]));
    kt.collect(S.ms_kernel, S.n_kernel);
    kt.on = false;
    std::lock_guard<std::mutex> lk(ctx->mu);
    hb_stats& T = ctx->stats;
    T.ms_consensus += ms;
    T.kernel_launches += launches;
    for (int i = 0; i < HB_NUM_KERNEL_CLASSES; i++) { T.ms_kernel[i] += S.ms_kernel[i]; T.n_kernel[i] += S.n_kernel[i]; }
    return HB_OK;
}

// ---------------------------------------------------------------------------------- hb_features_batch / hb_features_fetch
// The work of hb_features_batch, with the lane's lock held and the context's device current
int features_batch(hb_ctx* ctx, uint32_t n_targets, const uint32_t* rids, const uint32_t* n_ovl, const hb_overlap* ovl,
                   hb_features_shape* shape) {
    hb_ctx::FeatLane& Fl = ctx->feat;
    FeatResult& R = Fl.res;
    R.valid = false;  // the regions may move below
    if (!shape || (n_targets && (!rids || !n_ovl))) return fail(ctx, HB_ERR_ARG, "null pointer");
    if (!ctx->have_reads) return fail(ctx, HB_ERR_STATE, "hb_upload_reads must be called before hb_features_batch");
    uint64_t n_all = 0;
    for (uint32_t i = 0; i < n_targets; i++) n_all += n_ovl[i];
    if (n_all && !ovl) return fail(ctx, HB_ERR_ARG, "null pointer");
    const uint32_t W = ctx->opt.window_size, bs = ctx->opt.batch_size;
    // ---- every target prepared as hb_submit_alignments prepares it; coordinates the reference would panic on fail that target alone
    HostBatch& hbt = Fl.hbt;
    hbt.clear();
    R.status.assign(n_targets, HB_OK);
    R.n_windows.resize(n_targets);
    thread_local PreparedTarget P;
    std::string first_err;
    const hb_overlap* o = ovl;
    for (uint32_t i = 0; i < n_targets; i++) {
        const int rc = prepare_alignments(ctx, rids[i], o, n_ovl[i], P);
        if (rc == HB_ERR_INPUT) {
            R.status[i] = HB_ERR_INPUT;
            if (first_err.empty()) first_err = "target " + std::to_string(rids[i]) + ": " + errref(ctx);
        } else if (rc) {
            errref(ctx) = "target " + std::to_string(i) + " (rid " + std::to_string(rids[i]) + "): " + errref(ctx);
            return rc;
        } else {
            const int ra = append_target(ctx, hbt, P, o, n_ovl[i]);
            if (ra) return ra;
        }
        R.n_windows[i] = (ctx->read_len[rids[i]] + W - 1) / W;
        o += n_ovl[i];
    }
    // ---- the front half of a launch on the lane
    hb_ctx::Lane* L = &Fl.lane;
    const size_t nt = hbt.tgt.size(), nw = hbt.win.size();
    BatchView b{};
    Readback h{};
    uint64_t launches = 0, total_rows = 0;
    hb_stats S{};
    double t_wait = 0, t_mark = now_ms();
    float ms_front = 0;
    if (nt) {
        GatherSizes gs;
        ReadsInArgs g;
        int rc = run_front(ctx, L, hbt, b, h, &launches, &total_rows, gs, g, S, t_wait, t_mark);
        if (rc) { L->kt.discard(); return rc; }
        CK(Fl.pin_n1.grow(nw * 4));
        uint32_t* n1 = Fl.pin_n1.as<uint32_t>();
        CK(cudaMemcpyAsync(h.L, b.w_L, nw * 4, cudaMemcpyDeviceToHost, L->stream));
        CK(cudaMemcpyAsync(h.nsel, b.w_nsel, nw * 4, cudaMemcpyDeviceToHost, L->stream));
        CK(cudaMemcpyAsync(h.terr, b.tgt_err, nt * 4, cudaMemcpyDeviceToHost, L->stream));
        CK(cudaMemcpyAsync(n1, b.w_n1, nw * 4, cudaMemcpyDeviceToHost, L->stream));
        CK(cudaStreamSynchronize(L->stream));
        CK(cudaEventElapsedTime(&ms_front, L->ev[0], L->ev[2]));
        S.d2h_bytes = CNT_N * 4 + nw * 16 + nt * 4;
        L->kt.collect(S.ms_kernel, S.n_kernel);
        L->kt.on = false;
    }
    // ---- the caller's tables: windows of the targets in the given order, a failed target's without content
    R.rows.clear(); R.n_alns.clear(); R.n_sup.clear(); R.n_ids.clear(); R.dev_win.clear();
    R.batch_B.clear(); R.batch_Lmax.clear(); R.batch_win.clear();
    R.dev_rowbase.resize(nw);
    uint64_t rb = 0;
    for (size_t w = 0; w < nw; w++) { R.dev_rowbase[w] = rb; rb += h.L[w]; }
    hb_features_shape sh{};
    size_t t_dev = 0;  // the next target of the device batch
    uint32_t n_failed = 0;
    const uint32_t* n1 = Fl.pin_n1.as<uint32_t>();
    for (uint32_t i = 0; i < n_targets; i++) {
        const uint32_t nwin = R.n_windows[i];
        const uint32_t w_out0 = (uint32_t)R.rows.size();
        uint32_t dw0 = ~0u;
        if (R.status[i] == HB_OK) {
            const DevTarget& tg = hbt.tgt[t_dev++];
            if (h.terr[t_dev - 1] & TERR_BAD_INPUT) R.status[i] = HB_ERR_INPUT;
            else if (h.terr[t_dev - 1] & TERR_TOO_MANY_COLS) R.status[i] = HB_ERR_CAPACITY;
            if (R.status[i] == HB_OK) dw0 = tg.win_begin;
            else if (first_err.empty())
                first_err = "target " + std::to_string(rids[i]) + ": " +
                            (R.status[i] == HB_ERR_INPUT ? std::string("input the reference would panic on (malformed CIGAR / window descriptor / query coordinates)")
                                                         : "more than " + std::to_string(MAX_COLS_HARD) + " overlap-windows in one window");
        }
        if (R.status[i] != HB_OK) n_failed++;
        for (uint32_t k = 0; k < nwin; k++) {
            const bool ok = dw0 != ~0u;
            const uint32_t dw = ok ? dw0 + k : ~0u;
            R.dev_win.push_back(dw);
            R.rows.push_back(ok ? h.L[dw] : 0);
            R.n_alns.push_back(ok ? (uint8_t)h.nsel[dw] : 0);
            R.n_sup.push_back(ok ? h.nsup[dw] : 0);
            R.n_ids.push_back(ok ? n1[dw] : 0);
        }
        // the reference batches: groups of -b windows in wid order, of which the windows with supported positions (k_ref_lmax)
        for (uint32_t g0 = 0; g0 < nwin; g0 += bs) {
            uint32_t B = 0, lmax = 0;
            for (uint32_t k = g0; k < std::min(g0 + bs, nwin); k++)
                if (R.n_sup[w_out0 + k]) { R.batch_win.push_back(w_out0 + k); B++; lmax = std::max(lmax, R.rows[w_out0 + k]); }
            if (!B) continue;
            R.batch_B.push_back(B);
            R.batch_Lmax.push_back(lmax);
            sh.n_batch_rows += (uint64_t)B * lmax;
        }
    }
    for (size_t w = 0; w < R.rows.size(); w++) { sh.n_rows += R.rows[w]; sh.n_sup += R.n_sup[w]; sh.n_ids += R.n_ids[w]; }
    if (R.rows.size() >= (1ull << 32) || sh.n_sup >= (1ull << 32)) return fail(ctx, HB_ERR_CAPACITY, "batch too large: 2^32 windows or positions");
    sh.ticket = ++Fl.ticket;
    sh.n_targets = n_targets;
    sh.n_windows = (uint32_t)R.rows.size();
    sh.n_batches = (uint32_t)R.batch_B.size();
    sh.n_failed = n_failed;
    R.shape = sh;
    R.view = b;
    R.valid = true;
    *shape = sh;
    std::lock_guard<std::mutex> lk(ctx->mu);
    hb_stats& T = ctx->stats;
    T.ms_features += ms_front;
    T.kernel_launches += launches;
    T.h2d_bytes += S.h2d_bytes;
    T.d2h_bytes += S.d2h_bytes;
    for (int i = 0; i < HB_NUM_KERNEL_CLASSES; i++) { T.ms_kernel[i] += S.ms_kernel[i]; T.n_kernel[i] += S.n_kernel[i]; }
    if (!first_err.empty()) ctx->err = first_err;
    return HB_OK;
}

// The work of hb_features_fetch, with the lane's lock held and the context's device current
int features_fetch(hb_ctx* ctx, const hb_features_shape* shape, const hb_features_out* out, uint32_t flags, void* stream) {
    hb_ctx::FeatLane& Fl = ctx->feat;
    const FeatResult& R = Fl.res;
    if (!shape || !out) return fail(ctx, HB_ERR_ARG, "null pointer");
    if (out->struct_size != sizeof(hb_features_out)) return fail(ctx, HB_ERR_ARG, "hb_features_out.struct_size mismatch");
    if (flags & ~HB_FEAT_DEVICE_PTRS) return fail(ctx, HB_ERR_ARG, "unknown flags");
    if (!R.valid || shape->ticket != R.shape.ticket) return fail(ctx, HB_ERR_STATE, "the shape is not the context's latest hb_features_batch result");
    const bool dev = (flags & HB_FEAT_DEVICE_PTRS) != 0;
    {
        const void* p[15] = {out->bases, out->quals, out->batch_bases, out->batch_quals, out->status, out->n_windows, out->rows, out->n_alns,
                             out->n_sup, out->n_ids, out->supported, out->indices, out->ids, out->batch_B, out->batch_Lmax};
        static const char* name[15] = {"bases", "quals", "batch_bases", "batch_quals", "status", "n_windows", "rows", "n_alns", "n_sup",
                                       "n_ids", "supported", "indices", "ids", "batch_B", "batch_Lmax"};
        for (int i = 0; i < 16; i++) {
            const void* q = i < 15 ? p[i] : out->batch_win;
            if (!q) continue;
            const int k = pointer_kind(q, ctx->device);
            const char* nm = i < 15 ? name[i] : "batch_win";
            if (dev && i < 4 && k != 1)
                return fail(ctx, HB_ERR_ARG, std::string(nm) + " is not memory of device " + std::to_string(ctx->device) + " (HB_FEAT_DEVICE_PTRS is set)");
            if ((!dev || i >= 4) && k != 0)
                return fail(ctx, HB_ERR_ARG, std::string(nm) + " is device memory" + (i < 4 ? " (HB_FEAT_DEVICE_PTRS is not set)" : ""));
        }
    }
    const hb_features_shape& sh = R.shape;
    const size_t nt = sh.n_targets, nw = sh.n_windows;
    // ---- the metadata, from the host tables
    if (out->status && nt) memcpy(out->status, R.status.data(), nt * 4);
    if (out->n_windows && nt) memcpy(out->n_windows, R.n_windows.data(), nt * 4);
    if (out->rows && nw) memcpy(out->rows, R.rows.data(), nw * 4);
    if (out->n_alns && nw) memcpy(out->n_alns, R.n_alns.data(), nw);
    if (out->n_sup && nw) memcpy(out->n_sup, R.n_sup.data(), nw * 4);
    if (out->n_ids && nw) memcpy(out->n_ids, R.n_ids.data(), nw * 4);
    if (out->batch_B && sh.n_batches) memcpy(out->batch_B, R.batch_B.data(), (size_t)sh.n_batches * 4);
    if (out->batch_Lmax && sh.n_batches) memcpy(out->batch_Lmax, R.batch_Lmax.data(), (size_t)sh.n_batches * 4);
    if (out->batch_win && !R.batch_win.empty()) memcpy(out->batch_win, R.batch_win.data(), R.batch_win.size() * 4);
    const bool want_rows = (out->bases || out->quals) && sh.n_rows, want_batch = (out->batch_bases || out->batch_quals) && sh.n_batch_rows;
    const bool want_lists = ((out->supported || out->indices) && sh.n_sup) || (out->ids && sh.n_ids);
    if (!want_rows && !want_batch && !want_lists) return HB_OK;
    // ---- the tables of the output kernels: the ragged rows, the batch slots, the lists
    const BatchView& b = R.view;
    size_t n_rseg = 0, n_bseg = 0, n_lseg = 0;
    for (size_t w = 0; w < nw; w++) {
        if (R.rows[w]) n_rseg++;
        if (R.n_sup[w] || R.n_ids[w]) n_lseg++;
    }
    n_bseg = R.batch_win.size();
    Carve ct{nullptr};
    RowSeg *t_rows, *t_batch;
    ListSeg* t_lists;
    ct(t_rows, n_rseg); ct(t_batch, n_bseg); ct(t_lists, n_lseg);
    const size_t tab_bytes = ct.bytes;
    CK(Fl.pin_tab.grow(tab_bytes));
    CK(Fl.d_tab.grow(tab_bytes));
    Carve hc{Fl.pin_tab.as<uint8_t>()}, dc{Fl.d_tab.as<uint8_t>()};
    RowSeg *h_rows, *h_batch, *d_rows, *d_batch;
    ListSeg *h_lists, *d_lists;
    hc(h_rows, n_rseg); hc(h_batch, n_bseg); hc(h_lists, n_lseg);
    dc(d_rows, n_rseg); dc(d_batch, n_bseg); dc(d_lists, n_lseg);
    {
        uint64_t orow = 0, osup = 0, oid = 0;
        size_t kr = 0, kl = 0;
        for (size_t w = 0; w < nw; w++) {
            const uint32_t dw = R.dev_win[w];
            if (R.rows[w]) h_rows[kr++] = RowSeg{orow, R.dev_rowbase[dw], R.rows[w], R.rows[w]};
            if (R.n_sup[w] || R.n_ids[w]) h_lists[kl++] = ListSeg{dw, 0, osup, oid};
            orow += R.rows[w]; osup += R.n_sup[w]; oid += R.n_ids[w];
        }
        uint64_t brow = 0;
        size_t ks = 0;
        for (size_t k = 0; k < R.batch_B.size(); k++) {
            for (uint32_t s = 0; s < R.batch_B[k]; s++, ks++) {
                const uint32_t w = R.batch_win[ks];
                h_batch[ks] = RowSeg{brow + (uint64_t)s * R.batch_Lmax[k], R.dev_rowbase[R.dev_win[w]], R.rows[w], R.batch_Lmax[k]};
            }
            brow += (uint64_t)R.batch_B[k] * R.batch_Lmax[k];
        }
    }
    // ---- where the kernels write: the caller's device memory, or the staging region the host-bound outputs are copied from
    uint8_t *o_b = nullptr, *o_q = nullptr, *o_bb = nullptr, *o_bq = nullptr;
    uint32_t *o_sup = nullptr, *o_ids = nullptr;
    int32_t* o_idx = nullptr;
    {
        const size_t rb = want_rows ? sh.n_rows * R_COLS : 0, bb = want_batch ? sh.n_batch_rows * R_COLS : 0;
        Carve oc{nullptr};
        uint8_t *s_b, *s_q, *s_bb, *s_bq;
        uint32_t *s_sup, *s_ids;
        int32_t* s_idx;
        auto lay = [&](Carve& c) {
            c(s_b, dev || !out->bases ? 0 : rb); c(s_q, dev || !out->quals ? 0 : rb);
            c(s_bb, dev || !out->batch_bases ? 0 : bb); c(s_bq, dev || !out->batch_quals ? 0 : bb);
            c(s_sup, out->supported ? sh.n_sup * 2 : 0); c(s_idx, out->indices ? sh.n_sup : 0); c(s_ids, out->ids ? sh.n_ids : 0);
        };
        lay(oc);
        CK(Fl.d_out.grow(oc.bytes));
        Carve c{Fl.d_out.as<uint8_t>()};
        lay(c);
        o_b = !out->bases || !want_rows ? nullptr : dev ? out->bases : s_b;
        o_q = !out->quals || !want_rows ? nullptr : dev ? out->quals : s_q;
        o_bb = !out->batch_bases || !want_batch ? nullptr : dev ? out->batch_bases : s_bb;
        o_bq = !out->batch_quals || !want_batch ? nullptr : dev ? out->batch_quals : s_bq;
        o_sup = out->supported && sh.n_sup ? s_sup : nullptr;
        o_idx = out->indices && sh.n_sup ? s_idx : nullptr;
        o_ids = out->ids && sh.n_ids ? s_ids : nullptr;
    }
    // ---- device work
    hb_ctx::Lane* L = &Fl.lane;
    KTimer& kt = L->kt;
    kt.discard();
    kt.on = ctx->time_kernels.load(std::memory_order_relaxed);
    kt.st = L->stream;
    if (dev) {
        CK(cudaEventRecord(L->ev[3], (cudaStream_t)stream));
        CK(cudaStreamWaitEvent(L->stream, L->ev[3], 0));
    }
    CK(cudaMemcpyAsync(Fl.d_tab.p, Fl.pin_tab.p, tab_bytes, cudaMemcpyHostToDevice, L->stream));
    CK(cudaEventRecord(L->ev[4], L->stream));
    uint64_t launches = 0;
    if (o_b || o_q) { kt.begin(K_LISTS); launch_rows_out(d_rows, (uint32_t)n_rseg, b.mat_bases, b.mat_quals, o_b, o_q, L->stream); kt.end(); launches++; }
    if (o_bb || o_bq) { kt.begin(K_LISTS); launch_rows_out(d_batch, (uint32_t)n_bseg, b.mat_bases, b.mat_quals, o_bb, o_bq, L->stream); kt.end(); launches++; }
    if (o_sup || o_idx || o_ids) { kt.begin(K_LISTS); launch_lists_out(b, d_lists, (uint32_t)n_lseg, o_sup, o_idx, o_ids, L->stream); kt.end(); launches++; }
    CK(cudaGetLastError());
    CK(cudaEventRecord(L->ev[5], L->stream));
    // ---- host-bound outputs straight into the caller's memory
    uint64_t d2h = 0;
    auto copy = [&](void* dst, const void* src, size_t bytes) -> int {
        if (!dst || !src || !bytes) return HB_OK;
        CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, L->stream));
        d2h += bytes;
        return HB_OK;
    };
    int rc = HB_OK;
    if (!dev) {
        if (!rc) rc = copy(out->bases, o_b, sh.n_rows * R_COLS);
        if (!rc) rc = copy(out->quals, o_q, sh.n_rows * R_COLS);
        if (!rc) rc = copy(out->batch_bases, o_bb, sh.n_batch_rows * R_COLS);
        if (!rc) rc = copy(out->batch_quals, o_bq, sh.n_batch_rows * R_COLS);
    }
    if (!rc) rc = copy(out->supported, o_sup, sh.n_sup * 8);
    if (!rc) rc = copy(out->indices, o_idx, sh.n_sup * 4);
    if (!rc) rc = copy(out->ids, o_ids, sh.n_ids * 4);
    if (rc) { kt.discard(); return rc; }
    CK(cudaStreamSynchronize(L->stream));
    // ---- counters
    hb_stats S{};
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, L->ev[4], L->ev[5]));
    kt.collect(S.ms_kernel, S.n_kernel);
    kt.on = false;
    std::lock_guard<std::mutex> lk(ctx->mu);
    hb_stats& T = ctx->stats;
    T.ms_features += ms;
    T.kernel_launches += launches;
    T.h2d_bytes += tab_bytes;
    T.d2h_bytes += d2h;
    for (int i = 0; i < HB_NUM_KERNEL_CLASSES; i++) { T.ms_kernel[i] += S.ms_kernel[i]; T.n_kernel[i] += S.n_kernel[i]; }
    return HB_OK;
}

// ---------------------------------------------------------------------------------- read store
// ln(k) table from the host libm — the value Rust's f64::ln returns (src/features.rs:507)
int upload_ln_table(hb_ctx* ctx, uint32_t max_len) {
    ctx->ln_n = max_len + 2;
    std::vector<double> ln(ctx->ln_n);
    ln[0] = 0.0;
    for (uint32_t k = 1; k < ctx->ln_n; k++) ln[k] = std::log((double)k);
    CK(ctx->d_ln.grow((size_t)ctx->ln_n * 8));
    CK(cudaMemcpy(ctx->d_ln.p, ln.data(), (size_t)ctx->ln_n * 8, cudaMemcpyHostToDevice));
    return HB_OK;
}

// Leave the host store (lock held, context idle).  The lanes' last launches would gather from it again when replayed: they are
// dropped, and the context has no reads until the caller's upload or attach completes.
void detach_store(hb_ctx* ctx) {
    ctx->store->attached.fetch_sub(1);
    ctx->store = nullptr;
    ctx->store_words = nullptr;
    ctx->store_qual = nullptr;
    ctx->have_reads = false;
    for (auto& L : ctx->lanes) L.last.valid = false;
    ctx->last_lane = -1;
}

}  // namespace

// ========================================================================================
extern "C" {

int hb_inspect_model(const char* model_path, uint32_t dims[6], uint64_t* params_hash, char* err, size_t err_cap) {
    if (!model_path || !dims) return HB_ERR_ARG;
    uint32_t d9[9];
    const int rc = hb_inspect_model_ex(model_path, d9, params_hash, err, err_cap);
    if (rc == HB_OK) memcpy(dims, d9, 6 * sizeof(uint32_t));
    return rc;
}

int hb_inspect_model_ex(const char* model_path, uint32_t dims[9], uint64_t* params_hash, char* err, size_t err_cap) {
    if (!model_path || !dims) return HB_ERR_ARG;
    ModelFile mf;
    std::string e;
    const int rc = read_model_file(model_path, mf, e);
    if (rc != HB_OK) {
        if (err && err_cap) { strncpy(err, e.c_str(), err_cap - 1); err[err_cap - 1] = 0; }
        return rc;
    }
    for (int i = 0; i < 6; i++) dims[i] = mf.cfg[3 + i];
    for (int i = 0; i < 3; i++) dims[6 + i] = mf.cfg[10 + i];
    if (params_hash) {  // FNV-1a over the canonical tensors in name order: equal for a blob and an archive of the same weights
        uint64_t h = 1469598103934665603ull;
        for (auto& kv : mf.T) {
            for (unsigned char c : kv.first) { h ^= c; h *= 1099511628211ull; }
            const uint8_t* p = (const uint8_t*)kv.second.data();
            for (size_t i = 0; i < kv.second.size() * 4; i++) { h ^= p[i]; h *= 1099511628211ull; }
        }
        *params_hash = h;
    }
    return HB_OK;
}

const char* hb_last_error(hb_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

int hb_create(hb_ctx** out, int cuda_device, const char* model_path, const hb_options* opt) {
    const bool no_model = opt && opt->struct_size == sizeof(hb_options) && (opt->flags & HB_FLAG_NO_MODEL);
    if (!out || (!model_path && !no_model)) { g_create_err = "null argument"; return HB_ERR_ARG; }
    *out = nullptr;
    hb_ctx* ctx = new hb_ctx();
    ctx->device = cuda_device;
    ctx->opt.struct_size = sizeof(hb_options);
    ctx->opt.window_size = 4096;
    ctx->opt.batch_size = 64;
    ctx->opt.launch_targets = 256;
    ctx->opt.flags = 0;
    if (opt) {
        if (opt->struct_size != sizeof(hb_options)) { g_create_err = "hb_options.struct_size mismatch"; delete ctx; return HB_ERR_ARG; }
        if (opt->window_size) ctx->opt.window_size = opt->window_size;
        if (opt->batch_size) ctx->opt.batch_size = opt->batch_size;
        if (opt->launch_targets) ctx->opt.launch_targets = opt->launch_targets;
        ctx->opt.flags = opt->flags;
    }
    auto bail = [&](int code) { g_create_err = ctx->err; hb_destroy(ctx); return code; };
    if (ctx->opt.window_size < 8 || ctx->opt.window_size > 8192) { ctx->err = "window_size must be in [8, 8192]"; return bail(HB_ERR_ARG); }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        ctx->err = "no CUDA device: herro_b200 has no CPU fallback";
        return bail(HB_ERR_CUDA);
    }
    if (cuda_device < 0 || cuda_device >= ndev) { ctx->err = "cuda_device out of range"; return bail(HB_ERR_ARG); }
    if (cudaSetDevice(cuda_device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return bail(HB_ERR_CUDA); }
    if (const char* e = getenv("HERRO_B200_CHUNK_POS")) ctx->chunk_pos = (uint32_t)std::min(std::max(atoi(e), 128), 65536);
    if (const char* e = getenv("HERRO_B200_LANES")) ctx->n_lanes = std::min(std::max(atoi(e), 1), (int)hb_ctx::MAX_LANES);
    if (const char* e = getenv("HERRO_B200_MIN_LAUNCH")) ctx->min_launch = (uint32_t)std::min(std::max(atoi(e), 16), 4096);
    // debugging aids / A-B parity tests: read here once, never on the launch path
    ctx->pileup_v1 = getenv("HERRO_B200_PILEUP_V1") != nullptr;
    ctx->host_windowing = getenv("HERRO_B200_HOST_WINDOWING") != nullptr;
    if (const char* e = getenv("HERRO_B200_ARENA_ROWS")) ctx->arena_rows_per_win = (uint32_t)std::max(atoi(e), 1);
    ctx->wt.no_fuse_ln = getenv("HERRO_B200_NO_FUSE_LN") != nullptr;
    ctx->wt.no_fuse_ffn = getenv("HERRO_B200_NO_FUSE_FFN") != nullptr;
    ctx->wt.no_fuse_attn = getenv("HERRO_B200_NO_FUSE_ATTN") != nullptr;
    ctx->wt.no_fuse_oproj = getenv("HERRO_B200_NO_FUSE_OPROJ") != nullptr;
    if (!getenv("HERRO_B200_NO_NUMA_BIND")) probe_numa(ctx);
    for (int li = 0; li < ctx->n_lanes; li++) {
        auto& L = ctx->lanes[li];
        if (cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking) != cudaSuccess) { ctx->err = "cudaStreamCreate failed"; return bail(HB_ERR_CUDA); }
        for (auto& e : L.ev)
            if (cudaEventCreate(&e) != cudaSuccess) { ctx->err = "cudaEventCreate failed"; return bail(HB_ERR_CUDA); }
        L.d_batch.st = L.d_rows.st = L.d_fwd.st = L.stream;
    }
    {
        auto& F = ctx->fwd;
        if (cudaStreamCreateWithFlags(&F.stream, cudaStreamNonBlocking) != cudaSuccess) { ctx->err = "cudaStreamCreate failed"; return bail(HB_ERR_CUDA); }
        for (auto& e : F.ev)
            if (cudaEventCreate(&e) != cudaSuccess) { ctx->err = "cudaEventCreate failed"; return bail(HB_ERR_CUDA); }
        F.d_in.st = F.d_mat.st = F.d_fwd.st = F.stream;
    }
    {
        auto& Cn = ctx->cons;
        if (cudaStreamCreateWithFlags(&Cn.stream, cudaStreamNonBlocking) != cudaSuccess) { ctx->err = "cudaStreamCreate failed"; return bail(HB_ERR_CUDA); }
        for (auto& e : Cn.ev)
            if (cudaEventCreate(&e) != cudaSuccess) { ctx->err = "cudaEventCreate failed"; return bail(HB_ERR_CUDA); }
        Cn.d_in.st = Cn.d_out.st = Cn.stream;
    }
    {
        auto& Fl = ctx->feat;
        auto& L = Fl.lane;
        if (cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking) != cudaSuccess) { ctx->err = "cudaStreamCreate failed"; return bail(HB_ERR_CUDA); }
        for (auto& e : L.ev)
            if (cudaEventCreate(&e) != cudaSuccess) { ctx->err = "cudaEventCreate failed"; return bail(HB_ERR_CUDA); }
        L.d_batch.st = L.d_rows.st = L.d_fwd.st = Fl.d_tab.st = Fl.d_out.st = L.stream;
        Fl.hbt = HostBatch(cuda_device);
    }
    {   // keep freed blocks in the pool instead of returning them to the driver at every synchronisation
        cudaMemPool_t pool;
        uint64_t keep = UINT64_MAX;
        if (cudaDeviceGetDefaultMemPool(&pool, cuda_device) == cudaSuccess)
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    if (features_configure(ctx->opt.window_size) != cudaSuccess) { ctx->err = "kernel attribute setup failed (not an sm_90a device?)"; return bail(HB_ERR_CUDA); }
    ctx->no_model = no_model;
    if (!no_model) {
        const int rc = load_weights(ctx, model_path);
        if (rc) return bail(rc);
    }
    ctx->generation = g_ctx_generation.fetch_add(1);
    for (int i = 0; i < ctx->n_lanes; i++) ctx->lanes[i].worker = std::thread(worker_main, ctx, i);
    *out = ctx;
    return HB_OK;
}

void hb_destroy(hb_ctx* ctx) {
    if (!ctx) return;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        ctx->stop = true;
    }
    ctx->cv_work.notify_all();
    for (auto& L : ctx->lanes) if (L.worker.joinable()) L.worker.join();
    cudaSetDevice(ctx->device);
    for (auto& L : ctx->lanes) if (L.stream) cudaStreamSynchronize(L.stream);
    if (ctx->fwd.stream) cudaStreamSynchronize(ctx->fwd.stream);
    if (ctx->cons.stream) cudaStreamSynchronize(ctx->cons.stream);
    if (ctx->feat.lane.stream) cudaStreamSynchronize(ctx->feat.lane.stream);
    for (void* p : ctx->weight_allocs) cudaFree(p);
    if (ctx->store) ctx->store->attached.fetch_sub(1);
    DevBuf* bufs[] = {&ctx->d_words, &ctx->d_word_off, &ctx->d_len, &ctx->d_qual, &ctx->d_qual_off, &ctx->d_ln};
    for (DevBuf* b : bufs) b->release();
    for (auto& L : ctx->lanes) L.release();
    ctx->fwd.release();
    ctx->cons.release();
    ctx->feat.release();
    ctx->pin_in.release();
    ctx->slots.clear();
    ctx->queue.clear();
    ctx->pool.clear();
    delete ctx;
}

int hb_upload_reads(hb_ctx* ctx, uint32_t n_reads, const uint64_t* const* seq_words, const uint32_t* seq_len,
                    const uint8_t* const* qual) {
    if (!ctx) return HB_ERR_ARG;
    std::unique_lock<std::mutex> lk(ctx->mu);
    ctx->cv_idle.wait(lk, [&] { return ctx->idle(); });
    for (auto& sl : ctx->slots)
        if (!sl->batch.tgt.empty()) return fail(ctx, HB_ERR_STATE, "hb_upload_reads with targets pending: call hb_flush first");
    if (!seq_words || !seq_len || !qual || n_reads == 0) return fail(ctx, HB_ERR_ARG, "null/empty read store");
    CK(cudaSetDevice(ctx->device));
    if (ctx->store) detach_store(ctx);
    std::vector<uint64_t> woff(n_reads + 1, 0), qoff(n_reads + 1, 0);
    uint32_t max_len = 0;
    for (uint32_t i = 0; i < n_reads; i++) {
        woff[i + 1] = woff[i] + ((uint64_t)seq_len[i] + 31) / 32;
        qoff[i + 1] = qoff[i] + seq_len[i];
        max_len = std::max(max_len, seq_len[i]);
        if (!seq_words[i] || !qual[i]) return fail(ctx, HB_ERR_ARG, "null read");
    }
    // Padded on both sides: packed 32-base extraction may touch a few words past a read, and the pileup kernel fetches the
    // 4 bases / 4 quality bytes of a row group as whole words that may start up to 7 bytes before a read (pileup.cu).
    constexpr size_t FRONT_WORDS = 32, FRONT_QUAL = 256;  // keeps both bases 256-byte aligned
    CK(ctx->d_words.grow((FRONT_WORDS + woff[n_reads] + 8) * 8));
    CK(cudaMemset(ctx->d_words.p, 0, FRONT_WORDS * 8));
    CK(cudaMemset(ctx->d_words.as<uint64_t>() + FRONT_WORDS + woff[n_reads], 0, 8 * 8));
    CK(ctx->d_qual.grow(FRONT_QUAL + qoff[n_reads] + 16));
    CK(cudaMemset(ctx->d_qual.p, 33, FRONT_QUAL));
    CK(cudaMemset(ctx->d_qual.as<uint8_t>() + FRONT_QUAL + qoff[n_reads], 33, 16));
    CK(ctx->d_word_off.grow((n_reads + 1) * 8));
    CK(ctx->d_qual_off.grow((n_reads + 1) * 8));
    CK(ctx->d_len.grow((size_t)n_reads * 4));
    // stage in pinned chunks
    const size_t CH = 64u << 20;
    CK(ctx->pin_in.grow(CH));
    uint8_t* pin = ctx->pin_in.as<uint8_t>();
    auto copy_stream = [&](auto getp, auto getn, uint8_t* dbase) -> int {
        size_t fill = 0, doff = 0;
        for (uint32_t i = 0; i < n_reads; i++) {
            const uint8_t* src = (const uint8_t*)getp(i);
            size_t n = getn(i), so = 0;
            while (so < n) {
                const size_t take = std::min(n - so, CH - fill);
                memcpy(pin + fill, src + so, take);
                fill += take; so += take;
                if (fill == CH) {
                    CK(cudaMemcpy(dbase + doff, pin, fill, cudaMemcpyHostToDevice));
                    doff += fill; fill = 0;
                }
            }
        }
        if (fill) CK(cudaMemcpy(dbase + doff, pin, fill, cudaMemcpyHostToDevice));
        return HB_OK;
    };
    int rc = copy_stream([&](uint32_t i) { return (const void*)seq_words[i]; },
                         [&](uint32_t i) { return (size_t)(((uint64_t)seq_len[i] + 31) / 32 * 8); }, ctx->d_words.as<uint8_t>() + FRONT_WORDS * 8);
    if (rc) return rc;
    rc = copy_stream([&](uint32_t i) { return (const void*)qual[i]; }, [&](uint32_t i) { return (size_t)seq_len[i]; },
                     ctx->d_qual.as<uint8_t>() + FRONT_QUAL);
    if (rc) return rc;
    CK(cudaMemcpy(ctx->d_word_off.p, woff.data(), (n_reads + 1) * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ctx->d_qual_off.p, qoff.data(), (n_reads + 1) * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ctx->d_len.p, seq_len, (size_t)n_reads * 4, cudaMemcpyHostToDevice));
    rc = upload_ln_table(ctx, max_len);
    if (rc) return rc;
    ctx->stats.h2d_bytes += woff[n_reads] * 8 + qoff[n_reads];
    ctx->n_reads = n_reads;
    ctx->read_len.assign(seq_len, seq_len + n_reads);
    ctx->rs = ReadStoreView{ctx->d_words.as<uint64_t>() + FRONT_WORDS, ctx->d_word_off.as<uint64_t>(), ctx->d_len.as<uint32_t>(),
                            ctx->d_qual.as<uint8_t>() + FRONT_QUAL, ctx->d_qual_off.as<uint64_t>(), n_reads};
    ctx->have_reads = true;
    return HB_OK;
}

int hb_read_store_create(hb_read_store** out, uint32_t n_reads, const uint64_t* const* seq_words, const uint32_t* seq_len,
                         const uint8_t* const* qual) {
    g_create_err.clear();
    if (!out || !seq_words || !seq_len || !qual || n_reads == 0) { g_create_err = "null/empty read store"; return HB_ERR_ARG; }
    *out = nullptr;
    for (uint32_t i = 0; i < n_reads; i++)
        if (!seq_words[i] || !qual[i]) { g_create_err = "null read"; return HB_ERR_ARG; }
    std::unique_ptr<hb_read_store> s(new hb_read_store());
    s->n_reads = n_reads;
    s->len.assign(seq_len, seq_len + n_reads);
    s->word_off.resize(n_reads);
    s->qual_off.resize(n_reads);
    uint64_t w = 0, q = 0;
    for (uint32_t i = 0; i < n_reads; i++) {
        s->word_off[i] = w;
        s->qual_off[i] = q;
        w += ((uint64_t)seq_len[i] + 63) / 64 * 2;
        q += ((uint64_t)seq_len[i] + 15) / 16 * 16;
        s->max_len = std::max(s->max_len, seq_len[i]);
    }
    s->words_bytes = w * 8;
    s->bytes = s->words_bytes + q;
    const cudaError_t e = cudaHostAlloc((void**)&s->block, std::max<uint64_t>(s->bytes, 16), cudaHostAllocPortable | cudaHostAllocMapped);
    if (e != cudaSuccess) {
        s->block = nullptr;
        g_create_err = std::string("cudaHostAlloc of the read store (") + std::to_string(s->bytes) + " bytes): " + cudaGetErrorString(e);
        return e == cudaErrorMemoryAllocation ? HB_ERR_CAPACITY : HB_ERR_CUDA;
    }
    // every read with its padding: zero words up to an even count, quality 33 up to a multiple of 16 (the uploaded store's pad values)
    uint64_t* words = (uint64_t*)s->block;
    uint8_t* quals = s->block + s->words_bytes;
    const hb_read_store& S = *s;
    auto copy = [&](uint32_t i0, uint32_t i1) {
        for (uint32_t i = i0; i < i1; i++) {
            const uint64_t nw = ((uint64_t)seq_len[i] + 31) / 32, sw = ((uint64_t)seq_len[i] + 63) / 64 * 2;
            memcpy(words + S.word_off[i], seq_words[i], nw * 8);
            memset(words + S.word_off[i] + nw, 0, (sw - nw) * 8);
            const uint64_t sq = ((uint64_t)seq_len[i] + 15) / 16 * 16;
            memcpy(quals + S.qual_off[i], qual[i], seq_len[i]);
            memset(quals + S.qual_off[i] + seq_len[i], 33, sq - seq_len[i]);
        }
    };
    const uint32_t nth = std::min<uint32_t>(std::max(1u, std::thread::hardware_concurrency()), std::min<uint32_t>(16u, n_reads));
    std::vector<std::thread> th;
    for (uint32_t t = 0; t < nth; t++) th.emplace_back(copy, (uint32_t)((uint64_t)n_reads * t / nth), (uint32_t)((uint64_t)n_reads * (t + 1) / nth));
    for (auto& t : th) t.join();
    *out = s.release();
    return HB_OK;
}

int hb_read_store_destroy(hb_read_store* store) {
    if (!store) { g_create_err = "null read store"; return HB_ERR_ARG; }
    if (store->attached.load()) { g_create_err = "the read store is still attached to a context"; return HB_ERR_STATE; }
    cudaFreeHost(store->block);
    delete store;
    return HB_OK;
}

int hb_attach_read_store(hb_ctx* ctx, hb_read_store* store) {
    if (!ctx) return HB_ERR_ARG;
    std::unique_lock<std::mutex> lk(ctx->mu);
    ctx->cv_idle.wait(lk, [&] { return ctx->idle(); });
    for (auto& sl : ctx->slots)
        if (!sl->batch.tgt.empty()) return fail(ctx, HB_ERR_STATE, "hb_attach_read_store with targets pending: call hb_flush first");
    if (!store) return fail(ctx, HB_ERR_ARG, "null read store");
    CK(cudaSetDevice(ctx->device));
    void* dp = nullptr;
    CK(cudaHostGetDevicePointer(&dp, store->block, 0));
    if (ctx->store) detach_store(ctx);
    // the uploaded store's HBM is what this mode gives back
    for (DevBuf* b : {&ctx->d_words, &ctx->d_word_off, &ctx->d_qual, &ctx->d_qual_off}) b->release();
    for (auto& L : ctx->lanes) L.last.valid = false;  // their views point into the freed store
    ctx->last_lane = -1;
    ctx->have_reads = false;
    const uint32_t n = store->n_reads;
    CK(ctx->d_len.grow((size_t)n * 4));
    CK(cudaMemcpy(ctx->d_len.p, store->len.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
    const int rc = upload_ln_table(ctx, store->max_len);
    if (rc) return rc;
    ctx->stats.h2d_bytes += (uint64_t)n * 4 + (uint64_t)ctx->ln_n * 8;
    store->attached.fetch_add(1);
    ctx->store = store;
    ctx->store_words = (const uint64_t*)dp;
    ctx->store_qual = (const uint8_t*)dp + store->words_bytes;
    ctx->n_reads = n;
    ctx->read_len = store->len;
    ctx->rs = ReadStoreView{nullptr, nullptr, ctx->d_len.as<uint32_t>(), nullptr, nullptr, n};
    ctx->have_reads = true;
    return HB_OK;
}

int hb_submit_target(hb_ctx* ctx, uint32_t rid, uint32_t n_windows, const hb_overlap* ovl, uint32_t n_ovl,
                     const hb_overlap_window* ow, uint32_t n_ow) {
    if (!ctx) return HB_ERR_ARG;
    if (ctx->no_model) return no_model_fail(ctx);
    thread_local PreparedTarget P;  // its vectors keep their capacity from target to target
    P.raw = false;
    t_err_sink = nullptr;
    std::string local_err;
    {   // validation errors are written to a local string first: ctx->err is shared between feature threads
        t_err_sink = &local_err;
        const int rc = prepare_target(ctx, rid, n_windows, ovl, n_ovl, ow, n_ow, P);
        t_err_sink = nullptr;
        if (rc) { std::lock_guard<std::mutex> lk(ctx->mu); ctx->err = local_err; return rc; }
    }
    return stage_target(ctx, P, ovl, n_ovl);
}

int hb_submit_alignments(hb_ctx* ctx, uint32_t rid, const hb_overlap* ovl, uint32_t n_ovl) {
    if (!ctx) return HB_ERR_ARG;
    if (ctx->no_model) return no_model_fail(ctx);
    thread_local PreparedTarget P;  // scratch reused across calls
    std::string local_err;  // validation errors are written to a local string first: ctx->err is shared between feature threads
    t_err_sink = &local_err;
    const int rc = prepare_alignments(ctx, rid, ovl, n_ovl, P);
    t_err_sink = nullptr;
    if (rc) { std::lock_guard<std::mutex> lk(ctx->mu); ctx->err = local_err; return rc; }
    return stage_target(ctx, P, ovl, n_ovl);
}

int hb_extract_windows(const hb_overlap* ovl, uint32_t n_ovl, uint32_t window_size, uint32_t n_windows,
                       hb_overlap_window* out, uint32_t cap, uint32_t* n_out) {
    if ((!ovl && n_ovl) || !n_out || window_size == 0) return HB_ERR_ARG;
    std::vector<hb_overlap_window> v;
    for (uint32_t i = 0; i < n_ovl; i++)
        if (host_extract_windows(ovl[i], i, window_size, n_windows, v) != 0) return HB_ERR_INPUT;
    *n_out = (uint32_t)v.size();
    if (out) memcpy(out, v.data(), std::min<size_t>(v.size(), cap) * sizeof(hb_overlap_window));
    return HB_OK;
}

int hb_window_range(const hb_overlap* ovl, uint32_t window_size, uint32_t n_windows, uint32_t* first_window, uint32_t* end_window) {
    if (!ovl || !first_window || !end_window || window_size == 0) return HB_ERR_ARG;
    return skeleton_for_alignment(*ovl, window_size, n_windows, *first_window, *end_window) == 0 ? HB_OK : HB_ERR_INPUT;
}

int hb_set_launch_targets(hb_ctx* ctx, uint32_t launch_targets) {
    if (!ctx || launch_targets == 0) return HB_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->opt.launch_targets = launch_targets;
    return HB_OK;
}

int hb_set_kernel_timing(hb_ctx* ctx, int on) {
    if (!ctx) return HB_ERR_ARG;
    ctx->time_kernels.store(on != 0);
    return HB_OK;
}

int hb_flush(hb_ctx* ctx) {
    if (!ctx) return HB_ERR_ARG;
    if (ctx->no_model) return no_model_fail(ctx);
    std::unique_lock<std::mutex> lk(ctx->mu);
    {
        const uint32_t lt = ctx->opt.launch_targets, ns = std::max<uint32_t>(1u, (uint32_t)ctx->slots.size());
        const uint32_t full = ns >= 2 ? std::min(std::min(lt, std::max(ctx->min_launch, lt / ns)), 1024u) : 0u;
        for (auto& sl : ctx->slots) enqueue_batch(ctx, lk, sl->batch, full);  // must not race with hb_submit_* (see header)
    }
    ctx->handed_total.store(0);
    ctx->slots.clear();                                  // slots of finished feature threads are dropped;
    ctx->n_slots.store(0);
    ctx->generation = g_ctx_generation.fetch_add(1);    // live threads re-register on their next submit
    ctx->cv_idle.wait(lk, [&] { return ctx->idle(); });
    const int rc = ctx->worker_rc;
    if (rc != HB_OK) { ctx->err = ctx->worker_err; ctx->worker_rc = HB_OK; }
    return rc;
}

// Result block handed to the caller: [seg_len: n_segs u32, padded to 16][tag: u64 distance back to the block start,
// u64 magic][seq bytes].  hb_release_result finds the block from the tag in front of `seqs`, so neither call needs a
// table (or the context lock while copying).
static constexpr uint64_t RESULT_MAGIC = 0x4842524553303031ull;

int hb_poll_corrected(hb_ctx* ctx, uint32_t* rid, uint8_t** seqs, uint32_t** seg_len, uint32_t* n_segs) {
    if (!ctx || !rid || !seqs || !seg_len || !n_segs) return HB_ERR_ARG;
    Result r;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->results.empty()) return 0;
        r = std::move(ctx->results.front());
        ctx->results.pop_front();
    }
    *rid = r.rid;
    *seqs = nullptr;
    *seg_len = nullptr;
    *n_segs = 0;
    if (r.status != HB_OK) {  // nothing is allocated for a failed target: there is nothing to release
        std::lock_guard<std::mutex> lk(ctx->mu);
        ctx->err = "target " + std::to_string(r.rid) + ": " + r.msg;
        return r.status;
    }
    const size_t ns = r.seg_len.size();
    const size_t hdr = ((ns * 4 + 15) & ~(size_t)15) + 16;
    uint8_t* blk = (uint8_t*)malloc(hdr + r.seq.size() + 16);
    if (!blk) { std::lock_guard<std::mutex> lk(ctx->mu); return fail(ctx, HB_ERR_CAPACITY, "out of host memory"); }
    memcpy(blk, r.seg_len.data(), ns * 4);
    const uint64_t tag[2] = {(uint64_t)hdr, RESULT_MAGIC};
    memcpy(blk + hdr - 16, tag, 16);
    memcpy(blk + hdr, r.seq.data(), r.seq.size());
    *seg_len = (uint32_t*)blk;
    *seqs = blk + hdr;
    *n_segs = (uint32_t)ns;
    return 1;
}

int hb_bind_calling_thread(hb_ctx* ctx) {
    if (!ctx) return HB_ERR_ARG;
    if (!ctx->have_node_cpus) return 0;
    return pthread_setaffinity_np(pthread_self(), sizeof(cpu_set_t), &ctx->node_cpus) == 0 ? 1 : 0;
}

void hb_release_result(hb_ctx* ctx, uint8_t* seqs) {
    if (!ctx || !seqs) return;
    uint64_t tag[2];
    memcpy(tag, seqs - 16, 16);
    if (tag[1] != RESULT_MAGIC) return;  // not a block of hb_poll_corrected
    free(seqs - tag[0]);
}

int hb_get_stats(hb_ctx* ctx, hb_stats* out) {
    if (!ctx || !out) return HB_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    *out = ctx->stats;
    out->host_allocs = g_allocs.load() - ctx->alloc_base[0];
    out->ms_host_alloc = (double)(g_alloc_ns.load() - ctx->alloc_base[1]) * 1e-6;
    out->ms_submit_wait = (double)(g_submit_wait_ns.load() - ctx->alloc_base[2]) * 1e-6;
    return HB_OK;
}
int hb_reset_stats(hb_ctx* ctx) {
    if (!ctx) return HB_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->stats = hb_stats{};
    ctx->alloc_base[0] = g_allocs.load(); ctx->alloc_base[1] = g_alloc_ns.load(); ctx->alloc_base[2] = g_submit_wait_ns.load();
    return HB_OK;
}

static int find_window(hb_ctx* ctx, uint32_t rid, uint32_t wid, uint32_t* w) {
    if (!(ctx->opt.flags & HB_FLAG_KEEP_DEBUG)) return fail(ctx, HB_ERR_STATE, "context was not created with HB_FLAG_KEEP_DEBUG");
    if (ctx->last_lane < 0 || !ctx->lanes[ctx->last_lane].last.valid) return fail(ctx, HB_ERR_STATE, "no launch yet");
    const LastLaunch& last = ctx->lanes[ctx->last_lane].last;
    auto it = last.index.find(((uint64_t)rid << 32) | wid);
    if (it == last.index.end()) return fail(ctx, HB_ERR_ARG, "window not part of the most recent launch");
    *w = it->second;
    return HB_OK;
}

int hb_debug_window_shape(hb_ctx* ctx, uint32_t rid, uint32_t wid, uint32_t* shape4) {
    if (!ctx || !shape4) return HB_ERR_ARG;
    std::unique_lock<std::mutex> lk(ctx->mu);
    ctx->cv_idle.wait(lk, [&] { return ctx->idle(); });
    uint32_t w;
    int rc = find_window(ctx, rid, wid, &w);
    if (rc) return rc;
    const LastLaunch& last = ctx->lanes[ctx->last_lane].last;
    shape4[0] = last.w_L[w];
    shape4[1] = last.w_nsel[w];
    shape4[2] = last.w_nsup[w];
    shape4[3] = 1;
    return HB_OK;
}

int hb_debug_dump_window(hb_ctx* ctx, uint32_t rid, uint32_t wid, uint8_t* bases, uint8_t* quals, uint32_t* supported,
                         uint32_t* sup_rows, float* info_logits, float* bases_logits) {
    if (!ctx) return HB_ERR_ARG;
    std::unique_lock<std::mutex> lk(ctx->mu);
    ctx->cv_idle.wait(lk, [&] { return ctx->idle(); });
    CK(cudaSetDevice(ctx->device));
    uint32_t w;
    int rc = find_window(ctx, rid, wid, &w);
    if (rc) return rc;
    hb_ctx::Lane* lane = &ctx->lanes[ctx->last_lane];
    const LastLaunch& ll = lane->last;
    const uint32_t L = ll.w_L[w], ns = ll.w_nsup[w];
    const uint64_t rb = ll.w_rowbase[w], sb = ll.w_supbase[w];
    std::vector<uint8_t> tmp((size_t)L * ROW_BYTES);
    for (int pass = 0; pass < 2; pass++) {
        uint8_t* dst = pass ? quals : bases;
        if (!dst || !L) continue;
        CK(cudaMemcpy(tmp.data(), (pass ? ll.view.mat_quals : ll.view.mat_bases) + rb * ROW_BYTES, tmp.size(), cudaMemcpyDeviceToHost));
        for (uint32_t r = 0; r < L; r++) memcpy(dst + (size_t)r * R_COLS, tmp.data() + (size_t)r * ROW_BYTES, R_COLS);
    }
    if (ns) {
        std::vector<uint32_t> t(ns);
        if (supported) {
            CK(cudaMemcpy(t.data(), ll.view.sup_pk + rb, (size_t)ns * 4, cudaMemcpyDeviceToHost));
            for (uint32_t k = 0; k < ns; k++) { supported[2 * k] = (t[k] >> 8) & 0xffffu; supported[2 * k + 1] = t[k] & 0xffu; }
        }
        if (sup_rows) CK(cudaMemcpy(sup_rows, ll.view.sup_row + rb, (size_t)ns * 4, cudaMemcpyDeviceToHost));
        if (info_logits) CK(cudaMemcpy(info_logits, ll.fwd.info + sb, (size_t)ns * 4, cudaMemcpyDeviceToHost));
        if (bases_logits) CK(cudaMemcpy(bases_logits, ll.fwd.logits + sb * 5, (size_t)ns * 20, cudaMemcpyDeviceToHost));
    }
    return HB_OK;
}

// ---- `herro features` dump (src/features.rs:724-764,806-839) ---------------------------------------------------------
// .npy v1.0 exactly as numpy writes it: magic, u16 header length, the dict, padded with spaces to a multiple of 64, '\n'.
static bool write_npy(const std::string& path, const std::string& descr, const std::string& shape, const void* data, size_t bytes) {
    std::string dict = "{'descr': " + descr + ", 'fortran_order': False, 'shape': " + shape + ", }";
    size_t total = 10 + dict.size() + 1;
    const size_t pad = (64 - total % 64) % 64;
    dict.append(pad, ' ');
    dict.push_back('\n');
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) return false;
    const unsigned char magic[8] = {0x93, 'N', 'U', 'M', 'P', 'Y', 1, 0};
    const uint16_t hl = (uint16_t)dict.size();
    bool ok = fwrite(magic, 1, 8, f) == 8 && fwrite(&hl, 2, 1, f) == 1 && fwrite(dict.data(), 1, dict.size(), f) == dict.size() &&
              (bytes == 0 || fwrite(data, 1, bytes, f) == bytes);
    ok = fclose(f) == 0 && ok;
    return ok;
}

int hb_dump_features(hb_ctx* ctx, uint32_t rid, const char* out_dir, const char* const* read_names) {
    if (!ctx || !out_dir || !read_names) return HB_ERR_ARG;
    std::unique_lock<std::mutex> lk(ctx->mu);
    ctx->cv_idle.wait(lk, [&] { return ctx->idle(); });
    CK(cudaSetDevice(ctx->device));
    if (rid >= ctx->n_reads || !read_names[rid]) return fail(ctx, HB_ERR_ARG, "rid out of range / unnamed read");
    uint32_t w0;
    int rc = find_window(ctx, rid, 0, &w0);
    if (rc) return rc;
    hb_ctx::Lane* lane = &ctx->lanes[ctx->last_lane];
    const LastLaunch& ll = lane->last;
    const uint32_t W = ctx->opt.window_size, n_windows = (ctx->read_len[rid] + W - 1) / W;
    const std::string dir = std::string(out_dir) + "/" + read_names[rid];
    {   // create_dir_all
        std::string acc;
        for (size_t i = 0; i <= dir.size(); i++) {
            if (i == dir.size() || dir[i] == '/') { if (!acc.empty()) mkdir(acc.c_str(), 0777); }
            if (i < dir.size()) acc.push_back(dir[i]);
        }
    }
    static const char ASCII[13] = "ACGT*acgt#..";  // BASES_MAP inverted (src/inference.rs:23-31)
    std::vector<uint8_t> tb, tq, feat;
    std::vector<uint32_t> pk, order;
    for (uint32_t wid = 0; wid < n_windows; wid++) {
        const uint32_t w = w0 + wid;
        if (w >= ll.win.size() || ll.win[w].rid != rid || ll.win[w].wid != wid) return fail(ctx, HB_ERR_STATE, "target is not whole in the most recent launch");
        const uint32_t L = ll.w_L[w], ns = ll.w_nsup[w];
        const uint64_t rb = ll.w_rowbase[w];
        tb.resize((size_t)L * ROW_BYTES); tq.resize((size_t)L * ROW_BYTES);
        if (L) {
            CK(cudaMemcpy(tb.data(), ll.view.mat_bases + rb * ROW_BYTES, tb.size(), cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(tq.data(), ll.view.mat_quals + rb * ROW_BYTES, tq.size(), cudaMemcpyDeviceToHost));
        }
        // features: [2, L', 31] u8 — plane 0 the ASCII bases, plane 1 the quality bytes
        feat.resize((size_t)2 * L * R_COLS);
        for (uint32_t r = 0; r < L; r++)
            for (int c = 0; c < R_COLS; c++) {
                feat[(size_t)r * R_COLS + c] = (uint8_t)ASCII[tb[(size_t)r * ROW_BYTES + c] < 12 ? tb[(size_t)r * ROW_BYTES + c] : 11];
                feat[(size_t)L * R_COLS + (size_t)r * R_COLS + c] = tq[(size_t)r * ROW_BYTES + c];
            }
        const std::string base = dir + "/" + std::to_string(wid);
        if (!write_npy(base + ".features.npy", "'|u1'", "(2, " + std::to_string(L) + ", " + std::to_string(R_COLS) + ")", feat.data(), feat.size()))
            return fail(ctx, HB_ERR_ARG, "cannot write " + base + ".features.npy");
        // supported: 1-D array of SupportedPos {pos: u16, ins: u8}, packed (3 bytes per record)
        pk.resize(ns);
        if (ns) CK(cudaMemcpy(pk.data(), ll.view.sup_pk + rb, (size_t)ns * 4, cudaMemcpyDeviceToHost));
        std::vector<uint8_t> rec((size_t)ns * 3);
        for (uint32_t k = 0; k < ns; k++) {
            const uint16_t pos = (uint16_t)(pk[k] >> 8);
            memcpy(&rec[(size_t)k * 3], &pos, 2);
            rec[(size_t)k * 3 + 2] = (uint8_t)(pk[k] & 0xffu);
        }
        if (!write_npy(base + ".supported.npy", "[('pos', '<u2'), ('ins', '|u1')]", "(" + std::to_string(ns) + ",)", rec.data(), rec.size()))
            return fail(ctx, HB_ERR_ARG, "cannot write " + base + ".supported.npy");
        // ids: the query reads of ALL surviving overlaps of the window in final rank order (src/features.rs:569)
        uint32_t n1 = 0;
        CK(cudaMemcpy(&n1, ll.view.w_n1 + w, 4, cudaMemcpyDeviceToHost));
        order.resize(n1);
        if (n1) CK(cudaMemcpy(order.data(), ll.view.rank_ow + ll.win[w].ow_begin, (size_t)n1 * 4, cudaMemcpyDeviceToHost));
        FILE* f = fopen((base + ".ids.txt").c_str(), "wb");
        if (!f) return fail(ctx, HB_ERR_ARG, "cannot write " + base + ".ids.txt");
        for (uint32_t k = 0; k < n1; k++) {
            const uint32_t q = order[k] < ll.ow_qid.size() ? ll.ow_qid[order[k]] : 0;
            fprintf(f, "%s\n", q < ctx->n_reads && read_names[q] ? read_names[q] : "?");
        }
        fclose(f);
    }
    return HB_OK;
}

int hb_selftest_gemm(int cuda_device, uint32_t M, uint32_t N, uint32_t K, int act, int res, uint32_t lda_extra,
                     float* max_abs_err, float* max_abs_ref, float* ms_tc, float* ms_simt) {
    if (!max_abs_err || !max_abs_ref || M % 128 || N % 128 || K % 64 || (res && act && act != 3)) return HB_ERR_ARG;
    if (cudaSetDevice(cuda_device) != cudaSuccess) return HB_ERR_CUDA;
    const size_t lda = (size_t)K + lda_extra;
    std::vector<float> hA((size_t)M * lda), hW((size_t)N * K), hb(N), hR((size_t)M * N);
    uint64_t s = 0x9E3779B97F4A7C15ull;
    auto rnd = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return (float)((double)(s >> 11) / 9007199254740992.0 * 2.0 - 1.0); };
    for (auto& v : hA) v = rnd();
    for (auto& v : hW) v = rnd() * 0.1f;
    for (auto& v : hb) v = rnd();
    for (auto& v : hR) v = rnd();
    float *dA, *dW, *db, *dR, *dC1, *dC2;
    void *hi = nullptr, *lo = nullptr;
    bool ok = cudaMalloc(&dA, hA.size() * 4) == cudaSuccess && cudaMalloc(&dW, hW.size() * 4) == cudaSuccess &&
              cudaMalloc(&db, hb.size() * 4) == cudaSuccess && cudaMalloc(&dR, hR.size() * 4) == cudaSuccess &&
              cudaMalloc(&dC1, hR.size() * 4) == cudaSuccess && cudaMalloc(&dC2, hR.size() * 4) == cudaSuccess;
    if (!ok) return HB_ERR_CUDA;
    cudaMemcpy(dA, hA.data(), hA.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dW, hW.data(), hW.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(db, hb.data(), hb.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dR, hR.data(), hR.size() * 4, cudaMemcpyHostToDevice);
    if (split_weights(dW, hW.size(), &hi, &lo) != cudaSuccess) return HB_ERR_CUDA;
    void *ahi = nullptr, *alo = nullptr, *ohi = nullptr, *olo = nullptr;
    if (split_weights(dA, hA.size(), &ahi, &alo) != cudaSuccess) return HB_ERR_CUDA;
    if (cudaMalloc(&ohi, hR.size() * 2) != cudaSuccess || cudaMalloc(&olo, hR.size() * 2) != cudaSuccess) return HB_ERR_CUDA;
    int num_sms = 132;
    cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, cuda_device);
    GemmArgs ga{};
    ga.Ahi = (const __nv_bfloat16*)ahi; ga.Alo = (const __nv_bfloat16*)alo; ga.lda = lda;
    ga.Whi = (const __nv_bfloat16*)hi; ga.Wlo = (const __nv_bfloat16*)lo; ga.K = K;
    ga.bias = db; ga.out = dC2; ga.res = res ? dR : nullptr; ga.ldc = N;
    ga.out_hi = (__nv_bfloat16*)ohi; ga.out_lo = (__nv_bfloat16*)olo; ga.ldo = N;
    ga.m_tiles = M / 128; ga.n_chunks = N / 128; ga.k_blocks = K / 64;
    ga.mode = res ? GEMM_OUT_F32_RES : (act == 2 ? GEMM_OUT_SPLIT_RELU : (act ? GEMM_OUT_F32_RELU : GEMM_OUT_F32));
    if (act == 3) {  // residual + fused LayerNorm epilogue (N must be 128); compares the fp32 residual-stream output
        if (N != 128) return HB_ERR_ARG;
        ga.mode = GEMM_OUT_F32_RES_LN; ga.res = dC2; ga.ln_g = db; ga.ln_b = db; res = 1; act = 0;
        cudaMemcpy(dC2, dR, hR.size() * 4, cudaMemcpyDeviceToDevice);
    }
    cudaEvent_t e0, e1, e2;
    cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventCreate(&e2);
    cudaError_t e = cudaSuccess;
    for (int rep = 0; rep < 2; rep++) {  // second repetition is the timed one
        if (ga.mode == GEMM_OUT_F32_RES_LN) cudaMemcpy(dC2, dR, hR.size() * 4, cudaMemcpyDeviceToDevice);  // in-place residual
        cudaEventRecord(e0);
        gemm_simt(act ? 1 : 0, res, dA, (int)lda, dW, db, dC1, (int)N, res ? dR : nullptr, M, (int)N, (int)K, 0);
        cudaEventRecord(e1);
        e = gemm_tc(ga, num_sms, 0);
        cudaEventRecord(e2);
        if (e != cudaSuccess) break;
        e = cudaDeviceSynchronize();
        if (e != cudaSuccess) break;
    }
    if (e == cudaSuccess && act == 2) {  // recombine the split output into dC2 for the comparison
        std::vector<uint16_t> h1(hR.size()), h2(hR.size());
        cudaMemcpy(h1.data(), ohi, h1.size() * 2, cudaMemcpyDeviceToHost);
        cudaMemcpy(h2.data(), olo, h2.size() * 2, cudaMemcpyDeviceToHost);
        std::vector<float> c(hR.size());
        for (size_t i = 0; i < c.size(); i++) {
            uint32_t a = (uint32_t)h1[i] << 16, b2 = (uint32_t)h2[i] << 16;
            float fa, fb;
            memcpy(&fa, &a, 4); memcpy(&fb, &b2, 4);
            c[i] = fa + fb;
        }
        cudaMemcpy(dC2, c.data(), c.size() * 4, cudaMemcpyHostToDevice);
    }
    int rc = HB_OK;
    if (e != cudaSuccess) {
        g_create_err = std::string("selftest: ") + cudaGetErrorString(e);
        rc = HB_ERR_CUDA;
    } else {
        std::vector<float> c1(hR.size()), c2(hR.size());
        cudaMemcpy(c1.data(), dC1, c1.size() * 4, cudaMemcpyDeviceToHost);
        cudaMemcpy(c2.data(), dC2, c2.size() * 4, cudaMemcpyDeviceToHost);
        float me = 0, mr = 0;
        for (size_t i = 0; i < c1.size(); i++) {
            float d = fabsf(c1[i] - c2[i]);
            if (!(d <= me)) me = d;  // NaN propagates
            mr = std::max(mr, fabsf(c1[i]));
        }
        *max_abs_err = me;
        *max_abs_ref = mr;
        if (ms_simt) cudaEventElapsedTime(ms_simt, e0, e1);
        if (ms_tc) cudaEventElapsedTime(ms_tc, e1, e2);
    }
    cudaFree(dA); cudaFree(dW); cudaFree(db); cudaFree(dR); cudaFree(dC1); cudaFree(dC2); cudaFree(hi); cudaFree(lo); cudaFree(ahi); cudaFree(alo); cudaFree(ohi); cudaFree(olo);
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(e2);
    return rc;
}

int hb_selftest_pos_attention(int cuda_device, const uint32_t* lens, uint32_t n_seq, uint32_t heads, uint32_t head_dim,
                              const float* qkv, float* out, float* ms) {
    if (!lens || !qkv || !out || heads == 0 || (head_dim != 32 && head_dim != 64)) return HB_ERR_ARG;
    if (cudaSetDevice(cuda_device) != cudaSuccess) return HB_ERR_CUDA;
    const size_t D = (size_t)heads * head_dim;
    std::vector<uint64_t> base(n_seq);
    uint64_t rows = 0;
    for (uint32_t i = 0; i < n_seq; i++) { base[i] = rows; rows += lens[i]; }
    const size_t r1 = std::max<uint64_t>(rows, 1), s1 = std::max<uint32_t>(n_seq, 1);
    float* dq = nullptr;
    uint64_t* db = nullptr;
    uint32_t* dl = nullptr;
    __nv_bfloat16 *ohi = nullptr, *olo = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    cudaError_t e = cudaMalloc(&dq, r1 * 3 * D * 4);
    if (e == cudaSuccess) e = cudaMalloc(&db, s1 * 8);
    if (e == cudaSuccess) e = cudaMalloc(&dl, s1 * 4);
    if (e == cudaSuccess) e = cudaMalloc(&ohi, r1 * D * 2);
    if (e == cudaSuccess) e = cudaMalloc(&olo, r1 * D * 2);
    if (e == cudaSuccess) e = cudaMemcpy(dq, qkv, rows * 3 * D * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && n_seq) e = cudaMemcpy(db, base.data(), n_seq * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && n_seq) e = cudaMemcpy(dl, lens, n_seq * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(ohi, 0, r1 * D * 2);
    if (e == cudaSuccess) e = cudaMemset(olo, 0, r1 * D * 2);
    if (e == cudaSuccess) {
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        // the launcher of the forward's position-axis stage (forward.cu), on one chunk holding every sequence
        const PosAttnArgs pa{dq, 3 * D, db, dl, 0, n_seq, (int)D, (int)heads, ohi, olo, D};
        cudaEventRecord(e0);
        e = pos_attention(pa, 0);
        cudaEventRecord(e1);
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
    }
    if (e == cudaSuccess) {
        std::vector<uint16_t> h1(rows * D), h2(rows * D);
        e = cudaMemcpy(h1.data(), ohi, h1.size() * 2, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(h2.data(), olo, h2.size() * 2, cudaMemcpyDeviceToHost);
        for (size_t i = 0; e == cudaSuccess && i < h1.size(); i++) {
            const uint32_t a = (uint32_t)h1[i] << 16, b2 = (uint32_t)h2[i] << 16;
            float fa, fb;
            memcpy(&fa, &a, 4); memcpy(&fb, &b2, 4);
            out[i] = fa + fb;
        }
        if (e == cudaSuccess && ms) cudaEventElapsedTime(ms, e0, e1);
    }
    if (e != cudaSuccess) g_create_err = std::string("selftest: ") + cudaGetErrorString(e);
    cudaFree(dq); cudaFree(db); cudaFree(dl); cudaFree(ohi); cudaFree(olo);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    return e == cudaSuccess ? HB_OK : HB_ERR_CUDA;
}

int hb_replay_last_launch(hb_ctx* ctx, uint32_t iters, float* ms) {
    if (!ctx || !ms) return HB_ERR_ARG;
    std::unique_lock<std::mutex> lk(ctx->mu);
    ctx->cv_idle.wait(lk, [&] { return ctx->idle(); });
    CK(cudaSetDevice(ctx->device));
    if (ctx->last_lane < 0 || !ctx->lanes[ctx->last_lane].last.valid) return fail(ctx, HB_ERR_STATE, "no launch to replay");
    hb_ctx::Lane* L = &ctx->lanes[ctx->last_lane];
    const BatchView b = L->last.view;
    uint64_t launches = 0;
    L->kt.on = false;
    L->kt.st = L->stream;
    CK(cudaStreamSynchronize(L->stream));
    CK(cudaEventRecord(L->ev[6], L->stream));
    for (uint32_t it = 0; it < iters; it++) {
        int rc = zero_scratch(ctx, L, b);
        if (rc) return rc;
        if (L->last.gs.n_reads) launches += launch_reads_in(L->last.gather, L->stream, L->kt);
        launches += launch_features_a(b, L->stream, L->kt);
        launches += launch_pileup(b, L->stream, L->kt, ctx->pileup_v1);
        launches += launch_features_c1(b, L->stream, L->kt);
        rc = launch_tail(ctx, L, b, L->last.fwd, L->last.w_nsup.data(), L->last.w_nsup.size(), &launches);
        if (rc) return rc;
    }
    CK(cudaEventRecord(L->ev[7], L->stream));
    CK(cudaStreamSynchronize(L->stream));
    CK(cudaEventElapsedTime(ms, L->ev[6], L->ev[7]));
    L->kt.discard();
    ctx->stats.kernel_launches += launches;
    return HB_OK;
}

int hb_forward_batch(hb_ctx* ctx, uint32_t B, uint32_t Lmax, const uint8_t* bases, const uint8_t* quals, const int32_t* lens,
                     const int32_t* indices, float* info_logits, float* bases_logits, uint32_t flags, void* stream) {
    if (!ctx) return HB_ERR_ARG;
    if (ctx->no_model) return no_model_fail(ctx);
    std::lock_guard<std::mutex> lk(ctx->fwd.mu);
    int prev = -1;
    cudaGetDevice(&prev);
    std::string err;  // written to ctx->err under the context lock: the pipeline's threads share it
    t_err_sink = &err;
    int rc = cudaSetDevice(ctx->device) == cudaSuccess ? HB_OK : fail(ctx, HB_ERR_CUDA, "cudaSetDevice failed");
    if (rc == HB_OK) rc = forward_batch(ctx, B, Lmax, bases, quals, lens, indices, info_logits, bases_logits, flags, stream);
    t_err_sink = nullptr;
    if (prev >= 0 && prev != ctx->device) cudaSetDevice(prev);
    if (rc != HB_OK) {
        std::lock_guard<std::mutex> g(ctx->mu);
        ctx->err = err;
    }
    return rc;
}

int hb_consensus_batch(hb_ctx* ctx, uint32_t n_reads, const uint32_t* n_windows, const uint32_t* rows, const uint8_t* n_alns,
                       const uint8_t* bases, const uint32_t* n_sup, const uint32_t* supported, const float* bases_logits, uint8_t* seqs,
                       uint32_t* seg_len, uint32_t* n_segs, uint32_t flags, void* stream) {
    if (!ctx) return HB_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->cons.mu);
    int prev = -1;
    cudaGetDevice(&prev);
    std::string err;  // written to ctx->err under the context lock: the pipeline's threads share it
    t_err_sink = &err;
    int rc = cudaSetDevice(ctx->device) == cudaSuccess ? HB_OK : fail(ctx, HB_ERR_CUDA, "cudaSetDevice failed");
    if (rc == HB_OK)
        rc = consensus_batch(ctx, n_reads, n_windows, rows, n_alns, bases, n_sup, supported, bases_logits, seqs, seg_len, n_segs, flags,
                             stream);
    t_err_sink = nullptr;
    if (prev >= 0 && prev != ctx->device) cudaSetDevice(prev);
    if (rc != HB_OK) {
        std::lock_guard<std::mutex> g(ctx->mu);
        ctx->err = err;
    }
    return rc;
}

int hb_features_batch(hb_ctx* ctx, uint32_t n_targets, const uint32_t* rids, const uint32_t* n_ovl, const hb_overlap* ovl,
                      hb_features_shape* shape) {
    if (!ctx) return HB_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->feat.mu);
    int prev = -1;
    cudaGetDevice(&prev);
    std::string err;  // written to ctx->err under the context lock: the pipeline's threads share it
    t_err_sink = &err;
    int rc = cudaSetDevice(ctx->device) == cudaSuccess ? HB_OK : fail(ctx, HB_ERR_CUDA, "cudaSetDevice failed");
    if (rc == HB_OK) rc = features_batch(ctx, n_targets, rids, n_ovl, ovl, shape);
    t_err_sink = nullptr;
    if (prev >= 0 && prev != ctx->device) cudaSetDevice(prev);
    if (rc != HB_OK) {
        std::lock_guard<std::mutex> g(ctx->mu);
        ctx->err = err;
    }
    return rc;
}

int hb_features_fetch(hb_ctx* ctx, const hb_features_shape* shape, const hb_features_out* out, uint32_t flags, void* stream) {
    if (!ctx) return HB_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->feat.mu);
    int prev = -1;
    cudaGetDevice(&prev);
    std::string err;
    t_err_sink = &err;
    int rc = cudaSetDevice(ctx->device) == cudaSuccess ? HB_OK : fail(ctx, HB_ERR_CUDA, "cudaSetDevice failed");
    if (rc == HB_OK) rc = features_fetch(ctx, shape, out, flags, stream);
    t_err_sink = nullptr;
    if (prev >= 0 && prev != ctx->device) cudaSetDevice(prev);
    if (rc != HB_OK) {
        std::lock_guard<std::mutex> g(ctx->mu);
        ctx->err = err;
    }
    return rc;
}

}  // extern "C"
