// ks_api.cu — implementation of the C ABI declared in include/ksched.h (snapshot handle, staging,
// path selection).  Plain CUDA runtime; no torch, no oracle, no CPU fallback: every entry point that
// computes returns KS_ERR_NO_DEVICE / KS_ERR_CUDA when no H100 (sm_90) is present.
#include <cassert>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <condition_variable>
#include <deque>
#include <initializer_list>
#include <mutex>
#include <thread>
#include <algorithm>
#include <map>
#include <vector>

#include "ks_bitpar.h"
#include "ks_internal.cuh"
#include "ks_launch.h"

using namespace ks;

static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define CU_TRY(expr)                                                                                   \
    do {                                                                                               \
        cudaError_t _e = (expr);                                                                       \
        if (_e != cudaSuccess)                                                                         \
            return fail(KS_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                        __LINE__);                                                                     \
    } while (0)

struct ks_snapshot {
    int device = 0;
    Stream stream;
    uint32_t N = 0, Npad = 0, W = 1;
    DevBuf alloc_cpu, alloc_mem, free_cpu, free_mem, prio, labels, flag, xflag;
    // Staging shared by every call that holds mu until its final stream synchronise: no two are ever live, and the
    // snapshot keeps the largest any of them needed.  d_in: host-space pods and priorities, bound and claim lists
    // (CallerStaged) and the host-staged calls' inputs; d_out: every host-space result; d_work:
    // stream/gang, drain, scale-up and replica scratch; h_stage: the host-staged calls' pinned block (HostStaged).  A
    // call ensures each buffer once, for its whole layout, before it takes a pointer: a growing ensure frees those taken.
    HostBuf h_stage;
    DevBuf d_in, d_work, d_out;
    // Per call kind: an all-device select, top-k or preempt returns after enqueue and its kernels keep using these (as
    // they do the node table, flag, xflag and bp), so sharing one would let calls on two caller streams race.
    DevBuf part_sel, part_topk, part_pre, vx_pre; // node-chunk partials of select, top-k, preempt; preempt's victim index
    int sms = 0, coop = 0;
    Event ev[4];
    // host-space calls are pipelined in pod chunks: chunk c+1 is copied in on copy_stream while chunk c computes
    Stream copy_stream;
    Event ev_cfork, ev_in[4];
    bool timing_valid = false;
    bool derived_dirty = true; // prio + bit-parallel index must be rebuilt before the next select
    const char* last_path = "none";
    BitparIndex bp;
    // CUDA-graph replay of the launch sequence of an all-device ks_select (same arguments, same snapshot state)
    GraphExec graph_exec;
    uint64_t graph_key[16] = {0};
    bool graph_valid = false;
    uint64_t graph_launches = 0; // kernels inside the cached graph
    uint64_t version = 1; // bumped whenever device-side snapshot state or buffers change
    std::mutex mu;
};

static NodeTable node_table(ks_snapshot* s) {
    NodeTable nt;
    nt.free_cpu = s->free_cpu.as<int64_t>();
    nt.free_mem = s->free_mem.as<int64_t>();
    nt.alloc_cpu = s->alloc_cpu.as<int64_t>();
    nt.alloc_mem = s->alloc_mem.as<int64_t>();
    nt.labels = s->labels.as<uint64_t>();
    nt.N = s->N;
    nt.Npad = s->Npad;
    nt.W = s->W;
    return nt;
}

// free[] must stay inside the limits that keep scores in int64; prio[] = static node priority (KS_SCORE_LEFTOVER)
static int check_range_and_prio(ks_snapshot* s, cudaStream_t st) {
    if (s->N == 0) return KS_OK;
    CU_TRY(cudaMemsetAsync(s->flag.p, 0, sizeof(int), st));
    CU_TRY(launch_node_prio(s->free_cpu.as<int64_t>(), s->free_mem.as<int64_t>(), s->prio.as<int64_t>(), s->N, s->Npad,
                            s->flag.as<int>(), st));
    int flag = 0;
    CU_TRY(cudaMemcpyAsync(&flag, s->flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    if (flag) return fail(KS_ERR_RANGE, "free resources of some node exceed +-2^36 millicores / +-2^55 bytes");
    return KS_OK;
}

static bool valid_space(int32_t space) { return space == KS_MEM_HOST || space == KS_MEM_DEVICE; }
static bool valid_label_words(uint32_t W) { return W == 1 || W == 2 || W == 4 || W == 8; }
// inside +-2^36 millicores / +-2^55 bytes, the range that keeps every score inside int64
static bool within_limits(int64_t cpu, int64_t mem) {
    return cpu >= -KS_MAX_CPU_MILLI && cpu <= KS_MAX_CPU_MILLI && mem >= -KS_MAX_MEM_BYTES && mem <= KS_MAX_MEM_BYTES;
}

// Requests that are committed against free[] (claims, stream and gang pods) must lie in [0, limit]: an accepted claim
// then leaves its node's free in [0, free], so free[] stays inside the limits by construction.  Checked on the host
// before any device work.  (A negative request would always fit and raise free[]; API validation rejects them upstream.)
static int check_commit_requests(uint64_t n, const int64_t* req_cpu, const int64_t* req_mem) {
    for (uint64_t i = 0; i < n; i++)
        if (req_cpu[i] < 0 || req_cpu[i] > KS_MAX_CPU_MILLI || req_mem[i] < 0 || req_mem[i] > KS_MAX_MEM_BYTES)
            return fail(KS_ERR_RANGE, "pod %llu: request (%lld millicores, %lld bytes) outside [0, 2^36] / [0, 2^55]",
                        (unsigned long long)i, (long long)req_cpu[i], (long long)req_mem[i]);
    return KS_OK;
}

// ---- host-staged calls: ks_stream_bind's device loop, ks_gang_bind, ks_drain_check, ks_scaleup_estimate,
// ks_place_replicas, ks_place_replicas_spread (and _multi), and the bind walk's ks_spread_bind, ks_affinity_bind,
// ks_profile_bind, ks_node_bind, ks_fit_bind and ks_gang_fit_bind ----
// Such a call gathers its host inputs into the snapshot's pinned block, makes one H2D copy to d_in, launches, makes one
// D2H copy from d_out and copies its results out before it returns.  Its HostStaged plan declares every array it stages
// once, with its type and count: in() an input, gathered from src or, with src NULL, filled by the caller through
// host(); out() a result, copied to dst when dst is set and n > 0; work() device scratch in d_work.  The handle a
// declaration returns is the only way to the array afterwards, so its offset, size and type are written once.  The
// pinned block holds the inputs at 0 and the results at the next multiple of 16 after them.
// block: the plan's IN, OUT, WORK (or CallerStaged::CALLER); n elements.  A CallerStaged array also keeps its row width
// and the caller's pointer.
template <class T>
struct Staged { int block; size_t off; uint64_t n; uint64_t width = 1; T* caller = nullptr; };

class HostStaged {
  public:
    enum { IN, OUT, WORK };
    template <class T>
    Staged<T> in(const T* src, uint64_t n, size_t align = alignof(T)) { return add<T>(IN, const_cast<T*>(src), n, align); }
    template <class T>
    Staged<T> out(T* dst, uint64_t n, size_t align = alignof(T)) { return add<T>(OUT, dst, n, align); }
    template <class T>
    Staged<T> work(uint64_t n, size_t align = alignof(T)) { return add<T>(WORK, nullptr, n, align); }
    // With the snapshot locked and every array declared: ensures h_stage, d_in, d_out and d_work once, for the whole plan
    // and at least min_in / min_out bytes of inputs / results, then gathers the inputs that have a source.  A growing
    // ensure frees what the buffer held, so no pointer is handed out before this.  KS_OK or a KS_ERR_* with its message.
    int reserve(ks_snapshot* s, size_t min_in = 0, size_t min_out = 0) {
        if (overflow_)
            return fail(KS_ERR_RANGE, "a staging plan of more than %d gathered and scattered arrays", MAX_COPIES);
        const size_t in = std::max(layout_[IN].size, min_in), out = std::max(layout_[OUT].size, min_out);
        cudaError_t e = s->h_stage.ensure((in + 15) / 16 * 16 + out);
        if (e == cudaSuccess) e = s->d_in.ensure(in);
        if (e == cudaSuccess) e = s->d_out.ensure(out);
        if (e == cudaSuccess) e = s->d_work.ensure(layout_[WORK].size);
        if (e != cudaSuccess)
            return fail(KS_ERR_CUDA, "h.reserve(s) failed: %s (%s:%d)", cudaGetErrorString(e), __FILE__, __LINE__);
        dev_[IN] = s->d_in.p;
        dev_[OUT] = s->d_out.p;
        dev_[WORK] = s->d_work.p;
        host_[IN] = s->h_stage.p;
        host_[OUT] = at<unsigned char>(s->h_stage.p, (layout_[IN].size + 15) / 16 * 16);
        reserved_ = true;
        copy(IN);
        return cudaSuccess;
    }
    template <class T>
    T* dev(Staged<T> a) const {
        assert(reserved_);
        return at<T>(dev_[a.block], a.off);
    }
    // the pinned copy of an input or result: inputs before upload(), results after finish()
    template <class T>
    T* host(Staged<T> a) const {
        assert(reserved_ && a.block != WORK);
        return at<T>(host_[a.block], a.off);
    }
    cudaError_t upload(cudaStream_t st) const { // the one H2D copy
        return cudaMemcpyAsync(dev_[IN], host_[IN], layout_[IN].size, cudaMemcpyHostToDevice, st);
    }
    cudaError_t finish(cudaStream_t st) const { // the one D2H copy, a synchronise, then each result to its dst
        cudaError_t e = cudaMemcpyAsync(host_[OUT], dev_[OUT], layout_[OUT].size, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e == cudaSuccess) copy(OUT);
        return e;
    }

  private:
    struct Copy { int block; size_t off; void* p; size_t bytes; }; // p: an input's src or a result's dst
    template <class T>
    Staged<T> add(int block, T* p, uint64_t n, size_t align) {
        const size_t off = layout_[block].take<T>(n, align);
        if (p && n) {
            if (n_copies_ < MAX_COPIES) copies_[n_copies_++] = Copy{block, off, p, n * sizeof(T)};
            else overflow_ = true; // reported by reserve(), before any device work
        }
        return Staged<T>{block, off, n};
    }
    void copy(int block) const { // gathers the inputs into the pinned block, or scatters the results from it
        for (int i = 0; i < n_copies_; i++) {
            const Copy& c = copies_[i];
            if (c.block == IN && block == IN) memcpy(at<unsigned char>(host_[IN], c.off), c.p, c.bytes);
            if (c.block == OUT && block == OUT) memcpy(c.p, at<unsigned char>(host_[OUT], c.off), c.bytes);
        }
    }
    // The largest plan: ks_gang_fit_bind with every optional array given, 32 inputs and 8 results (bind_spread)
    static constexpr int MAX_COPIES = 40;
    BlockLayout layout_[3];
    void* dev_[3] = {};
    void* host_[2] = {};
    Copy copies_[MAX_COPIES];
    int n_copies_ = 0;
    bool overflow_ = false;
    bool reserved_ = false;
};

// The scratch of k_stream_batch and k_gang_batch in d_work, [pkey | pidx | pend] (the kernels rebuild the pending list on
// every call: nothing in it persists), declared on the caller's plan.
struct StreamBatchScratch { Staged<int64_t> key; Staged<int32_t> idx; Staged<uint32_t> pend; };
static StreamBatchScratch stream_batch_scratch(HostStaged& h, int sms) {
    return {h.work<int64_t>((size_t)STREAM_BATCH_MAX * sms), h.work<int32_t>((size_t)STREAM_BATCH_MAX * sms, 256),
            h.work<uint32_t>(2 * STREAM_BATCH_MAX, 256)};
}

// What k_stream_batch and k_gang_batch take from the snapshot: the node table, the policy, the grid and the scratch, after
// reserve().  The caller sets the pods, the outputs, ctl and max_rounds.
static StreamBatchArgs stream_batch_args(const ks_snapshot* s, int policy, const HostStaged& h, const StreamBatchScratch& w) {
    StreamBatchArgs a;
    a.N = s->N;
    a.Npad = s->Npad;
    a.alloc_cpu = s->alloc_cpu.as<int64_t>();
    a.alloc_mem = s->alloc_mem.as<int64_t>();
    a.labels = s->labels.as<uint64_t>();
    a.free_cpu = s->free_cpu.as<int64_t>();
    a.free_mem = s->free_mem.as<int64_t>();
    a.policy = policy;
    a.pkey = h.dev(w.key);
    a.pidx = h.dev(w.idx);
    a.pend = h.dev(w.pend);
    a.grid = std::max(1u, std::min<uint32_t>((uint32_t)s->sms, (s->N + 127u) / 128u));
    return a;
}

// ---- caller-space calls: ks_select, ks_select_topk, ks_explain, ks_preempt, ks_check_cells / ks_check_cell,
// ks_select_sampling, and the claim lists of set_bound, apply_bind and commit_claims ----
// The caller says per array whether it is in host or device memory, and every array is rows of a fixed width, one row
// per pod or claim.  Such a call declares each array once on a CallerStaged plan: in() an input, out() a result, work()
// node-chunk partials in the call kind's own buffer.  A host-space array gets a slot at a multiple of 256 bytes, an
// input in d_in and a result in d_out; a device-space array is used in place; an absent one (NULL) or one with no rows
// takes no space and no copy.  Unlike HostStaged's one gathered copy, upload() and download() copy each host-space array
// straight between the caller's memory, which may be pageable, and the device, on the call's stream, so a CUDA graph
// can capture them.
namespace { // file-local: none of its members is exported
class CallerStaged {
  public:
    enum { IN, OUT, WORK, CALLER }; // CALLER: used in place (device-space) or absent
    explicit CallerStaged(DevBuf* part = nullptr) : part_(part) {}
    template <class T>
    Staged<T> in(const T* src, uint64_t rows, uint64_t width, bool host) {
        return add<T>(host ? IN : CALLER, const_cast<T*>(src), rows, width, -1);
    }
    // clear() fills a result's bytes with empty
    template <class T>
    Staged<T> out(T* dst, uint64_t rows, uint64_t width, bool host, uint8_t empty = 0) {
        return add<T>(host ? OUT : CALLER, dst, rows, width, empty);
    }
    template <class T>
    Staged<T> work(uint64_t rows, uint64_t width) {
        assert(part_);
        return add<T>(WORK, nullptr, rows, width, -1);
    }
    // With the snapshot locked and every array declared: ensures d_in, d_out and the partial buffer once, for the whole
    // plan.  A growing ensure frees what the buffer held, so no pointer is handed out before this.
    cudaError_t reserve(ks_snapshot* s) {
        cudaError_t e = s->d_in.ensure(layout_[IN].size);
        if (e == cudaSuccess) e = s->d_out.ensure(layout_[OUT].size);
        if (e == cudaSuccess && part_) e = part_->ensure(layout_[WORK].size);
        if (e != cudaSuccess) return e;
        base_[IN] = s->d_in.p;
        base_[OUT] = s->d_out.p;
        base_[WORK] = part_ ? part_->p : nullptr;
        reserved_ = true;
        return cudaSuccess;
    }
    // the device array from row on; NULL when absent or empty
    template <class T>
    T* dev(Staged<T> a, uint64_t row = 0) const {
        assert(reserved_);
        T* p = a.block == CALLER ? a.caller : at<T>(base_[a.block], a.off);
        return a.n && p ? p + row * a.width : nullptr;
    }
    // the caller's host destination of a host-space result from row on; NULL otherwise
    template <class T>
    T* host(Staged<T> a, uint64_t row = 0) const {
        return a.block == OUT && a.n ? a.caller + row * a.width : nullptr;
    }
    cudaError_t upload(cudaStream_t st, uint64_t r0, uint64_t r1) const { // rows [r0, r1) of every host-space input
        for (int i = 0; i < n_arrays_; i++) {
            const Array& a = arrays_[i];
            if (a.block != IN || r1 == r0) continue;
            cudaError_t e = cudaMemcpyAsync(row(a, r0), a.caller + r0 * a.row_bytes, (r1 - r0) * a.row_bytes,
                                            cudaMemcpyHostToDevice, st);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    // rows [r0, r1) of every host-space result, except those whose destination (from r0 on) is in served: a launcher
    // copied them already
    cudaError_t download(cudaStream_t st, uint64_t r0, uint64_t r1, std::initializer_list<const void*> served = {}) const {
        for (int i = 0; i < n_arrays_; i++) {
            const Array& a = arrays_[i];
            unsigned char* dst = a.caller + r0 * a.row_bytes;
            if (a.block != OUT || r1 == r0 || std::find(served.begin(), served.end(), dst) != served.end()) continue;
            cudaError_t e = cudaMemcpyAsync(dst, row(a, r0), (r1 - r0) * a.row_bytes, cudaMemcpyDeviceToHost, st);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    cudaError_t clear(cudaStream_t st) const { // every result filled with its empty byte
        for (int i = 0; i < n_arrays_; i++) {
            const Array& a = arrays_[i];
            if (a.empty < 0) continue;
            cudaError_t e = cudaMemsetAsync(row(a, 0), a.empty, a.rows * a.row_bytes, st);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    bool any_host() const { return any_host_; } // then the call synchronises before it returns

  private:
    struct Array { int block; size_t off; unsigned char* caller; size_t row_bytes; uint64_t rows; int empty; };
    template <class T>
    Staged<T> add(int block, T* p, uint64_t rows, uint64_t width, int empty) {
        any_host_ |= block == IN || block == OUT;
        if (block != WORK && (!p || !rows)) return Staged<T>{CALLER, 0, 0, width, nullptr};
        const size_t off = block == CALLER ? 0 : layout_[block].take<T>(rows * width, 256);
        if (block != WORK) {
            assert(n_arrays_ < MAX_ARRAYS);
            arrays_[n_arrays_++] = Array{block, off, reinterpret_cast<unsigned char*>(p), width * sizeof(T), rows, empty};
        }
        return Staged<T>{block, off, rows * width, width, p};
    }
    unsigned char* row(const Array& a, uint64_t r) const {
        return (a.block == CALLER ? a.caller : at<unsigned char>(base_[a.block], a.off)) + r * a.row_bytes;
    }
    static constexpr int MAX_ARRAYS = 8;
    DevBuf* part_;
    BlockLayout layout_[3];
    void* base_[3] = {};
    Array arrays_[MAX_ARRAYS];
    int n_arrays_ = 0;
    bool any_host_ = false;
    bool reserved_ = false;
};

// The pods of a caller-space call, [rc | rm | sel]: one row per pod, sel W words wide.
struct StagedPods {
    Staged<int64_t> cpu, mem;
    Staged<uint64_t> sel;
    PodView view(const CallerStaged& plan, uint64_t r0, uint64_t r1) const {
        return PodView{plan.dev(cpu, r0), plan.dev(mem, r0), plan.dev(sel, r0), (uint32_t)(r1 - r0)};
    }
};
} // namespace
static StagedPods declare_pods(CallerStaged& plan, const ks_pods* pods, uint32_t W) {
    const bool host = pods->mem_space == KS_MEM_HOST;
    return {plan.in(pods->req_cpu, pods->n, 1, host), plan.in(pods->req_mem, pods->n, 1, host),
            plan.in(pods->sel, pods->n, W, host)};
}

// the caller's stream, or the snapshot's when the caller passes none
static cudaStream_t call_stream(const ks_snapshot* s, void* cuda_stream) {
    return cuda_stream ? (cudaStream_t)cuda_stream : s->stream.h;
}

extern "C" {

// internal hook for the host layer (host/ksh_host.cpp); not declared in include/
void ks__set_error(const char* msg) { snprintf(g_err, sizeof(g_err), "%s", msg ? msg : ""); }

const char* ks_last_error(void) { return g_err; }
int ks_version(void) { return 100; }
int ks_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}
uint64_t ks_launch_count(void) { return g_launches.load(); }
uint64_t ks_mask_row_bytes(uint32_t n_nodes) { return 32ull * ((n_nodes + 255ull) / 256ull); }
uint64_t ks_mask_row_bytes_aligned(uint32_t n_nodes) { return 256ull * ((n_nodes + 2047ull) / 2048ull); }

int ks_snapshot_create(int device, ks_snapshot** out) {
    if (!out) return fail(KS_ERR_INVALID, "out is NULL");
    *out = nullptr;
    int n = ks_device_count();
    if (n <= 0) return fail(KS_ERR_NO_DEVICE, "no CUDA device visible: libksched has no CPU fallback");
    if (device < 0 || device >= n) return fail(KS_ERR_INVALID, "device %d out of range [0,%d)", device, n);
    CU_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(KS_ERR_NO_DEVICE, "device %d is sm_%d%d; libksched is built for sm_90a only", device, prop.major,
                    prop.minor);
    ks_snapshot* s = new (std::nothrow) ks_snapshot();
    if (!s) return fail(KS_ERR_NOMEM, "out of host memory");
    s->device = device;
    s->sms = prop.multiProcessorCount;
    s->coop = prop.cooperativeLaunch;
    cudaError_t e = cudaStreamCreateWithFlags(&s->stream.h, cudaStreamNonBlocking);
    for (int i = 0; i < 4 && e == cudaSuccess; i++) e = cudaEventCreate(&s->ev[i].h);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->copy_stream.h, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->ev_cfork.h, cudaEventDisableTiming);
    for (int i = 0; i < 4 && e == cudaSuccess; i++) e = cudaEventCreateWithFlags(&s->ev_in[i].h, cudaEventDisableTiming);
    if (e == cudaSuccess) e = s->flag.ensure(sizeof(int));
    if (e == cudaSuccess) e = s->xflag.ensure(sizeof(int));
    if (e == cudaSuccess) e = cudaMemset(s->xflag.p, 0, sizeof(int));
    if (e == cudaSuccess) e = prepare_direct();
    if (e != cudaSuccess) {
        ks_snapshot_destroy(s);
        return fail(KS_ERR_CUDA, "snapshot init failed: %s", cudaGetErrorString(e));
    }
    *out = s;
    return KS_OK;
}

void ks_snapshot_destroy(ks_snapshot* s) {
    if (!s) return;
    cudaSetDevice(s->device);
    if (s->stream) cudaStreamSynchronize(s->stream);
    delete s; // frees the buffers and destroys the handles: the device is set and the stream synchronised
}

uint32_t ks_snapshot_num_nodes(const ks_snapshot* s) { return s ? s->N : 0; }
uint32_t ks_snapshot_label_words(const ks_snapshot* s) { return s ? s->W : 0; }

int ks_snapshot_set_nodes(ks_snapshot* s, uint32_t n_nodes, uint32_t label_words, const int64_t* alloc_cpu,
                          const int64_t* alloc_mem, const uint64_t* labels) {
    if (!s) return fail(KS_ERR_INVALID, "snapshot is NULL");
    if (!valid_label_words(label_words))
        return fail(KS_ERR_INVALID, "label_words must be 1, 2, 4 or 8 (got %u)", label_words);
    if (n_nodes && (!alloc_cpu || !alloc_mem || !labels)) return fail(KS_ERR_INVALID, "NULL node array");
    if (n_nodes > (1u << 30)) return fail(KS_ERR_RANGE, "n_nodes too large");
    for (uint32_t n = 0; n < n_nodes; n++)
        if (!within_limits(alloc_cpu[n], alloc_mem[n]))
            return fail(KS_ERR_RANGE, "node %u allocatable outside +-2^36 millicores / +-2^55 bytes", n);
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    const uint32_t Npad = ((n_nodes + TILE_N - 1) / TILE_N) * TILE_N;
    s->N = n_nodes;
    s->Npad = Npad;
    s->W = label_words;
    s->derived_dirty = true;
    s->version++;
    if (Npad == 0) return KS_OK;
    std::vector<int64_t> h;
    std::vector<uint64_t> hl;
    try { // no exception crosses the ABI
        h.resize(Npad);
        hl.assign((size_t)Npad * label_words, 0);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory staging %u nodes", n_nodes);
    }
    const size_t nb = (size_t)Npad * 8;
    CU_TRY(s->alloc_cpu.ensure(nb));
    CU_TRY(s->alloc_mem.ensure(nb));
    CU_TRY(s->free_cpu.ensure(nb));
    CU_TRY(s->free_mem.ensure(nb));
    CU_TRY(s->prio.ensure(2 * nb)); // [leftover priority | least-allocated bound]
    CU_TRY(s->labels.ensure(nb * label_words));
    // allocatable: pad with 0; free: pad with INT64_MIN (never feasible)
    for (uint32_t n = 0; n < Npad; n++) h[n] = n < n_nodes ? alloc_cpu[n] : 0;
    CU_TRY(cudaMemcpyAsync(s->alloc_cpu.p, h.data(), nb, cudaMemcpyHostToDevice, s->stream));
    for (uint32_t n = n_nodes; n < Npad; n++) h[n] = INT64_MIN;
    CU_TRY(cudaMemcpyAsync(s->free_cpu.p, h.data(), nb, cudaMemcpyHostToDevice, s->stream));
    CU_TRY(cudaStreamSynchronize(s->stream));
    for (uint32_t n = 0; n < Npad; n++) h[n] = n < n_nodes ? alloc_mem[n] : 0;
    CU_TRY(cudaMemcpyAsync(s->alloc_mem.p, h.data(), nb, cudaMemcpyHostToDevice, s->stream));
    for (uint32_t n = n_nodes; n < Npad; n++) h[n] = INT64_MIN;
    CU_TRY(cudaMemcpyAsync(s->free_mem.p, h.data(), nb, cudaMemcpyHostToDevice, s->stream));
    for (uint32_t n = 0; n < n_nodes; n++)
        for (uint32_t w = 0; w < label_words; w++) hl[(size_t)w * Npad + n] = labels[(size_t)n * label_words + w];
    CU_TRY(cudaMemcpyAsync(s->labels.p, hl.data(), nb * label_words, cudaMemcpyHostToDevice, s->stream));
    CU_TRY(cudaStreamSynchronize(s->stream));
    return check_range_and_prio(s, s->stream);
}

static int reset_free_to_alloc(ks_snapshot* s) {
    // free[0..N) = alloc[0..N); the padding keeps its INT64_MIN sentinels
    CU_TRY(cudaMemcpyAsync(s->free_cpu.p, s->alloc_cpu.p, (size_t)s->N * 8, cudaMemcpyDeviceToDevice, s->stream));
    CU_TRY(cudaMemcpyAsync(s->free_mem.p, s->alloc_mem.p, (size_t)s->N * 8, cudaMemcpyDeviceToDevice, s->stream));
    return KS_OK;
}

int ks_snapshot_set_bound(ks_snapshot* s, uint64_t n_bound, const int32_t* node_idx, const int64_t* req_cpu,
                          const int64_t* req_mem) {
    if (!s) return fail(KS_ERR_INVALID, "snapshot is NULL");
    if (n_bound && (!node_idx || !req_cpu || !req_mem)) return fail(KS_ERR_INVALID, "NULL bound array");
    for (uint64_t b = 0; b < n_bound; b++) {
        if (node_idx[b] < 0 || (uint32_t)node_idx[b] >= s->N)
            return fail(KS_ERR_INVALID, "bound pod %llu: node index %d out of range", (unsigned long long)b,
                        node_idx[b]);
        if (!within_limits(req_cpu[b], req_mem[b]))
            return fail(KS_ERR_RANGE, "bound pod %llu request out of range", (unsigned long long)b);
    }
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    s->derived_dirty = true;
    s->version++;
    if (s->N == 0) return KS_OK;
    int rc = reset_free_to_alloc(s);
    if (rc) return rc;
    if (n_bound) {
        CallerStaged plan;
        const auto node = plan.in(node_idx, n_bound, 1, true);
        const auto cpu = plan.in(req_cpu, n_bound, 1, true), mem = plan.in(req_mem, n_bound, 1, true);
        CU_TRY(plan.reserve(s));
        CU_TRY(plan.upload(s->stream, 0, n_bound));
        CU_TRY(launch_free_reduce(s->free_cpu.as<int64_t>(), s->free_mem.as<int64_t>(), plan.dev(node), plan.dev(cpu),
                                  plan.dev(mem), n_bound, s->stream));
    }
    return check_range_and_prio(s, s->stream);
}

int ks_snapshot_apply_bind(ks_snapshot* s, int32_t node_idx, int64_t req_cpu, int64_t req_mem) {
    if (!s) return fail(KS_ERR_INVALID, "snapshot is NULL");
    if (node_idx < 0 || (uint32_t)node_idx >= s->N) return fail(KS_ERR_INVALID, "node index %d out of range", node_idx);
    if (!within_limits(req_cpu, req_mem)) return fail(KS_ERR_RANGE, "request out of range");
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    // free[] stays inside the limits: refuse a bind that would take the node's free outside them, before anything
    // changes (both values are inside them, so the differences cannot overflow)
    int64_t f[2];
    CU_TRY(cudaMemcpyAsync(&f[0], s->free_cpu.as<int64_t>() + node_idx, 8, cudaMemcpyDeviceToHost, s->stream));
    CU_TRY(cudaMemcpyAsync(&f[1], s->free_mem.as<int64_t>() + node_idx, 8, cudaMemcpyDeviceToHost, s->stream));
    CU_TRY(cudaStreamSynchronize(s->stream));
    const int64_t nc = f[0] - req_cpu, nm = f[1] - req_mem;
    if (!within_limits(nc, nm))
        return fail(KS_ERR_RANGE, "node %d: the bind would leave free at %lld millicores / %lld bytes, outside +-2^36 / +-2^55",
                    node_idx, (long long)nc, (long long)nm);
    s->derived_dirty = true;
    s->version++;
    CallerStaged plan;
    const auto node = plan.in(&node_idx, 1, 1, true);
    const auto cpu = plan.in(&req_cpu, 1, 1, true), mem = plan.in(&req_mem, 1, 1, true);
    CU_TRY(plan.reserve(s));
    CU_TRY(plan.upload(s->stream, 0, 1));
    CU_TRY(launch_free_reduce(s->free_cpu.as<int64_t>(), s->free_mem.as<int64_t>(), plan.dev(node), plan.dev(cpu),
                              plan.dev(mem), 1, s->stream));
    CU_TRY(cudaStreamSynchronize(s->stream));
    return KS_OK;
}

int ks_snapshot_get_free(ks_snapshot* s, int64_t* free_cpu, int64_t* free_mem) {
    if (!s || !free_cpu || !free_mem) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    if (s->N == 0) return KS_OK;
    CU_TRY(cudaMemcpyAsync(free_cpu, s->free_cpu.p, (size_t)s->N * 8, cudaMemcpyDeviceToHost, s->stream));
    CU_TRY(cudaMemcpyAsync(free_mem, s->free_mem.p, (size_t)s->N * 8, cudaMemcpyDeviceToHost, s->stream));
    CU_TRY(cudaStreamSynchronize(s->stream));
    return KS_OK;
}

// rebuild what depends on free[]: range check, static priorities, bit-parallel index
static int refresh_derived(ks_snapshot* s, cudaStream_t st) {
    if (!s->derived_dirty || s->N == 0) return KS_OK;
    CU_TRY(launch_node_prio(s->free_cpu.as<int64_t>(), s->free_mem.as<int64_t>(), s->prio.as<int64_t>(), s->N, s->Npad,
                            s->flag.as<int>(), st));
    cudaError_t e = bitpar_build(s->bp, node_table(s), s->prio.as<int64_t>(), st);
    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "bit-parallel index build failed: %s", cudaGetErrorString(e));
    s->derived_dirty = false;
    s->version++;
    return KS_OK;
}

static bool is_pinned_host(const void* p) {
    if (!p) return true;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost;
}

static int check_pods(const ks_snapshot* s, const ks_pods* pods) {
    if (!s) return fail(KS_ERR_INVALID, "snapshot is NULL");
    if (!pods) return fail(KS_ERR_INVALID, "pods is NULL");
    if (pods->n > 0xfffffff0ull) return fail(KS_ERR_RANGE, "too many pods in one call");
    if (pods->n && (!pods->req_cpu || !pods->req_mem || !pods->sel)) return fail(KS_ERR_INVALID, "NULL pod array");
    if (!valid_space(pods->mem_space)) return fail(KS_ERR_INVALID, "bad pods.mem_space");
    return KS_OK;
}

int ks_check_cells(ks_snapshot* s, const ks_pods* pods, uint8_t* out_codes) {
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (!out_codes) return fail(KS_ERR_INVALID, "out_codes is NULL");
    const uint64_t cells = pods->n * (uint64_t)s->N;
    if (cells == 0) return KS_OK;
    if (cells > (1ull << 31)) return fail(KS_ERR_RANGE, "ks_check_cells is for <= 2^31 cells");
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    CallerStaged plan;
    const StagedPods pd = declare_pods(plan, pods, s->W);
    const auto codes = plan.out(out_codes, pods->n, s->N, true);
    CU_TRY(plan.reserve(s));
    CU_TRY(plan.upload(s->stream, 0, pods->n));
    CU_TRY(launch_check_cells(node_table(s), pd.view(plan, 0, pods->n), plan.dev(codes), 0, s->N, s->stream));
    CU_TRY(plan.download(s->stream, 0, pods->n));
    CU_TRY(cudaStreamSynchronize(s->stream));
    return KS_OK;
}

int ks_check_cell(ks_snapshot* s, int64_t req_cpu, int64_t req_mem, const uint64_t* sel, uint32_t node_idx) {
    if (!s || !sel) return fail(KS_ERR_INVALID, "NULL argument");
    if (node_idx >= s->N) return fail(KS_ERR_INVALID, "node index %u out of range", node_idx);
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    const ks_pods pods{1, &req_cpu, &req_mem, sel, KS_MEM_HOST};
    uint8_t code = 0xff;
    CallerStaged plan;
    const StagedPods pd = declare_pods(plan, &pods, s->W);
    const auto out = plan.out(&code, 1, 1, true);
    CU_TRY(plan.reserve(s));
    CU_TRY(plan.upload(s->stream, 0, 1));
    CU_TRY(launch_check_cells(node_table(s), pd.view(plan, 0, 1), plan.dev(out), node_idx, 1, s->stream));
    CU_TRY(plan.download(s->stream, 0, 1));
    CU_TRY(cudaStreamSynchronize(s->stream));
    return (int)code;
}

int ks_select(ks_snapshot* s, const ks_pods* pods, int policy, uint32_t flags, ks_bindings* out, void* cuda_stream) {
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (!out) return fail(KS_ERR_INVALID, "out is NULL");
    if (!policy_valid(policy)) return fail(KS_ERR_INVALID, "bad policy");
    if ((flags & KS_SELECT_FORCE_BITPAR) && (flags & KS_SELECT_FORCE_DIRECT)) return fail(KS_ERR_INVALID, "bad flags");
    const uint64_t P = pods->n;
    if (out->mask) {
        if (out->mask_row_bytes % 32 != 0 || out->mask_row_bytes < ks_mask_row_bytes(s->N))
            return fail(KS_ERR_INVALID, "mask_row_bytes must be a multiple of 32 and >= %llu",
                        (unsigned long long)ks_mask_row_bytes(s->N));
        if (out->mask_space == KS_MEM_DEVICE && ((uintptr_t)out->mask & 31u) != 0)
            return fail(KS_ERR_INVALID, "a device-space mask must be 32-byte aligned");
    }
    const ks_exchange* xc = out->exchange;
    if (xc) {
        if (out->mem_space != KS_MEM_DEVICE || !out->node_idx || !out->score)
            return fail(KS_ERR_INVALID, "exchange needs device-space node_idx and score outputs");
        if (xc->world < 2 || xc->world > KS_MAX_PEERS + 1 || xc->rank >= xc->world || xc->n_peers != xc->world - 1)
            return fail(KS_ERR_INVALID, "bad exchange world/rank/n_peers");
        if (!xc->local_flags || !xc->local_state) return fail(KS_ERR_INVALID, "exchange: NULL local_flags / local_state");
        for (uint32_t k = 0; k < xc->n_peers; k++)
            if (!xc->peer_node_idx[k] || !xc->peer_score[k] || !xc->peer_flag[k])
                return fail(KS_ERR_INVALID, "exchange: NULL peer pointer %u", k);
    }
    if (P == 0 && !xc) return KS_OK;
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    const cudaStream_t st = call_stream(s, cuda_stream);
    const bool timing = (flags & KS_SELECT_TIMING) != 0;
    PeerOut po;
    if (xc) {
        po.n = xc->n_peers;
        po.world = xc->world;
        po.rank = xc->rank;
        for (uint32_t k = 0; k < xc->n_peers; k++) {
            po.idx[k] = xc->peer_node_idx[k];
            po.score[k] = xc->peer_score[k];
            po.flag[k] = xc->peer_flag[k];
        }
        po.local_flags = xc->local_flags;
        po.state = xc->local_state;
    }
    if (P == 0) { // an empty shard still takes part in the exchange: publish the sequence number, wait for the others
        CU_TRY(launch_exchange_push(po, nullptr, nullptr, 0, st));
        CU_TRY(launch_exchange_wait(po, s->xflag.as<int>(), st));
        return KS_OK;
    }
    s->timing_valid = false;
    if (timing) CU_TRY(cudaEventRecord(s->ev[0], st));

    // the per-cell kernel needs no derived state; the bit-parallel index is (re)built lazily
    const bool may_bitpar = (flags & KS_SELECT_FORCE_BITPAR) ||
                            (!(flags & KS_SELECT_FORCE_DIRECT) && (uint64_t)P * s->N >= (1ull << 24));
    if (may_bitpar) {
        rc = refresh_derived(s, st);
        if (rc) return rc;
    }

    const bool out_host = out->mem_space == KS_MEM_HOST;
    const bool mask_host = out->mask && out->mask_space == KS_MEM_HOST;
    bool use_bitpar = false;
    DirectGrid grid{};
    if (s->N) {
        if (flags & KS_SELECT_FORCE_BITPAR) use_bitpar = true;
        else if (!(flags & KS_SELECT_FORCE_DIRECT))
            use_bitpar = may_bitpar && bitpar_profitable(s->bp, (uint32_t)P);
        if (!use_bitpar) grid = direct_grid(s->W, (uint32_t)P, s->Npad, s->sms);
    }
    // everything that allocates happens before the (possibly captured) launch sequence; with no node, no mask row is
    // written
    CallerStaged plan(&s->part_sel);
    const StagedPods pd = declare_pods(plan, pods, s->W);
    const auto idx = plan.out(out->node_idx, P, 1, out_host, 0xff);
    const auto score = plan.out(out->score, P, 1, out_host);
    const auto cnt = plan.out(out->feasible_cnt, P, 1, out_host);
    const auto mask = plan.out(reinterpret_cast<uint32_t*>(out->mask), s->N ? P : 0, out->mask_row_bytes / 4, mask_host);
    const uint64_t part_rows = grid.n_chunks > 1 ? (uint64_t)grid.n_chunks * P : 0; // keys | indices | counts
    const auto pkey = plan.work<int64_t>(part_rows, 1);
    const auto pidx = plan.work<int32_t>(part_rows, 1);
    const auto pcnt = plan.work<uint32_t>(part_rows, 1);
    if (use_bitpar) {
        cudaError_t e = bitpar_prepare(s->bp, (uint32_t)P);
        if (e == cudaSuccess) e = bitpar_prepare_order(s->bp, node_table(s), policy, st);
        if (e != cudaSuccess) return fail(KS_ERR_CUDA, "bit-parallel prepare failed: %s", cudaGetErrorString(e));
    }
    CU_TRY(plan.reserve(s));

    if (s->N == 0) { // empty node store: every pod gets None (src/main.rs:56,70)
        CU_TRY(plan.clear(st));
        if (xc) {
            CU_TRY(launch_exchange_push(po, plan.dev(idx), plan.dev(score), (uint32_t)P, st));
            CU_TRY(launch_exchange_wait(po, s->xflag.as<int>(), st));
        }
        CU_TRY(plan.download(st, 0, P));
        s->last_path = "empty";
    } else {
        SelectLaunch L;
        L.nt = node_table(s);
        L.policy = policy;
        L.stream = st;
        L.po = po;
        L.ready_event = out_host ? nullptr : (cudaEvent_t)out->bindings_ready_event;
        const PartialView part{plan.dev(pkey), plan.dev(pidx), plan.dev(pcnt)};
        s->last_path = use_bitpar ? "bitpar" : "direct";
        // Host-space batches on the bit-parallel path are pipelined in two pod chunks: the second chunk is copied in
        // on copy_stream while the first computes, and the bindings of a chunk travel back under the next chunk's
        // mask kernel.  (Each chunk is an independent select over its pod range; scratch is reused because a chunk
        // starts only after the previous chunk's auxiliary-stream work has joined.)  A single chunk is copied in on st.
        const uint32_t n_pipe = (use_bitpar && pods->mem_space == KS_MEM_HOST && out_host && !mask_host && !timing &&
                                 P >= 262144) // below that the per-chunk launch overhead outweighs the overlap (measured at 100k pods)
                                    ? 2u
                                    : 1u;
        auto enqueue = [&]() -> int {
            if (n_pipe > 1) {
                CU_TRY(cudaEventRecord(s->ev_cfork, st));
                CU_TRY(cudaStreamWaitEvent(s->copy_stream, s->ev_cfork, 0));
            }
            for (uint32_t c = 0; c < n_pipe; c++) {
                CU_TRY(plan.upload(n_pipe > 1 ? s->copy_stream.h : st, P * c / n_pipe, P * (c + 1) / n_pipe));
                if (n_pipe > 1) CU_TRY(cudaEventRecord(s->ev_in[c], s->copy_stream));
            }
            for (uint32_t c = 0; c < n_pipe; c++) {
                const uint64_t c0 = P * c / n_pipe, c1 = P * (c + 1) / n_pipe;
                if (n_pipe > 1) CU_TRY(cudaStreamWaitEvent(st, s->ev_in[c], 0));
                SelectLaunch Lc = L;
                Lc.pv = pd.view(plan, c0, c1);
                Lc.ov = OutView{plan.dev(idx, c0), plan.dev(score, c0), plan.dev(cnt, c0), plan.dev(mask, c0),
                                out->mask_row_bytes / 4, (uint32_t)(ks_mask_row_bytes(s->N) / 4)};
                // served early by the launcher when it can, which then clears them
                int32_t* const h_idx = Lc.host_node_idx = plan.host(idx, c0);
                int64_t* const h_score = Lc.host_score = plan.host(score, c0);
                if (use_bitpar) {
                    cudaError_t e = bitpar_select(s->bp, Lc, timing ? s->ev[1].h : nullptr, timing ? s->ev[2].h : nullptr);
                    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "bit-parallel select failed: %s", cudaGetErrorString(e));
                } else {
                    if (timing) CU_TRY(cudaEventRecord(s->ev[1], st));
                    cudaError_t e = launch_select_direct(Lc, part, grid);
                    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "direct select failed: %s", cudaGetErrorString(e));
                    if (timing) CU_TRY(cudaEventRecord(s->ev[2], st));
                    if (xc) CU_TRY(launch_exchange_push(po, Lc.ov.node_idx, Lc.ov.score, Lc.pv.P, st));
                }
                // fused all-gather: this rank's bindings went out from the argmax kernels (bit-parallel path) or the push
                // kernel; the call's stream work ends when every other rank's bindings have arrived here
                if (xc) CU_TRY(launch_exchange_wait(po, s->xflag.as<int>(), st));
                CU_TRY(plan.download(st, c0, c1, {Lc.host_node_idx ? nullptr : h_idx, Lc.host_score ? nullptr : h_score}));
                if (Lc.ready_event) { // not served earlier (per-cell path): the bindings are final here
                    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
                    CU_TRY(cudaStreamIsCapturing(st, &cs));
                    CU_TRY(cudaEventRecordWithFlags(Lc.ready_event, st, cs == cudaStreamCaptureStatusActive ? cudaEventRecordExternal
                                                                                                        : cudaEventRecordDefault));
                }
            }
            return KS_OK;
        };
        // Replay from a cached CUDA graph when the call repeats (same buffers, same snapshot state).  Host buffers
        // qualify only if they are pinned (a captured copy from pageable memory is not allowed).
        const uint64_t key[16] = {P, (uint64_t)pods->req_cpu, (uint64_t)pods->req_mem, (uint64_t)pods->sel,
                                  (uint64_t)out->node_idx, (uint64_t)out->score, (uint64_t)out->feasible_cnt,
                                  (uint64_t)out->mask, out->mask_row_bytes,
                                  (uint64_t)policy | ((uint64_t)pods->mem_space << 8) | ((uint64_t)out->mem_space << 9) |
                                      ((uint64_t)out->mask_space << 10),
                                  (uint64_t)flags ^ ((uint64_t)out->bindings_ready_event << 8) ^ ((uint64_t)(xc ? xc->local_state : nullptr) << 20), (uint64_t)st, s->version, (uint64_t)use_bitpar,
                                  g_devbuf_epoch.load()};
        const bool key_hit = s->graph_valid && memcmp(key, s->graph_key, sizeof(key)) == 0;
        bool graph_ok = !timing && !(flags & KS_SELECT_NO_GRAPH);
        if (graph_ok && !key_hit) {
            if (pods->mem_space == KS_MEM_HOST)
                graph_ok = is_pinned_host(pods->req_cpu) && is_pinned_host(pods->req_mem) && is_pinned_host(pods->sel);
            if (graph_ok && out_host)
                graph_ok = is_pinned_host(out->node_idx) && is_pinned_host(out->score) && is_pinned_host(out->feasible_cnt);
            if (graph_ok && mask_host) graph_ok = is_pinned_host(out->mask);
        }
        if (graph_ok) {
            if (!key_hit) {
                s->graph_exec.reset();
                s->graph_valid = false;
                CU_TRY(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
                const uint64_t launches_before = g_launches.load();
                const int erc = enqueue();
                s->graph_launches = g_launches.load() - launches_before; // captured, not executed yet
                g_launches -= s->graph_launches;
                Graph graph;
                cudaError_t e = cudaStreamEndCapture(st, &graph.h);
                if (erc) return erc;
                if (e != cudaSuccess) return fail(KS_ERR_CUDA, "stream capture failed: %s", cudaGetErrorString(e));
                e = cudaGraphInstantiate(&s->graph_exec.h, graph, 0);
                if (e != cudaSuccess) return fail(KS_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(e));
                memcpy(s->graph_key, key, sizeof(key));
                s->graph_valid = true;
            }
            CU_TRY(cudaGraphLaunch(s->graph_exec, st));
            g_launches += s->graph_launches;
        } else {
            rc = enqueue();
            if (rc) return rc;
        }
    }
    if (timing) {
        CU_TRY(cudaEventRecord(s->ev[3], st));
        s->timing_valid = s->N != 0;
    }
    if (plan.any_host() || timing) CU_TRY(cudaStreamSynchronize(st));
    return KS_OK;
}

int ks_last_timings(ks_snapshot* s, float ms[3]) {
    if (!s || !ms) return fail(KS_ERR_INVALID, "NULL argument");
    if (!s->timing_valid) return fail(KS_ERR_INVALID, "no KS_SELECT_TIMING call recorded");
    CU_TRY(cudaSetDevice(s->device));
    CU_TRY(cudaEventSynchronize(s->ev[3]));
    CU_TRY(cudaEventElapsedTime(&ms[0], s->ev[1], s->ev[2]));
    CU_TRY(cudaEventElapsedTime(&ms[1], s->ev[2], s->ev[3]));
    CU_TRY(cudaEventElapsedTime(&ms[2], s->ev[0], s->ev[3]));
    return KS_OK;
}

const char* ks_last_path(const ks_snapshot* s) { return s ? s->last_path : "none"; }

int ks_last_trace(ks_snapshot* s, uint64_t out_ns[16]) {
    if (!s || !out_ns) return fail(KS_ERR_INVALID, "NULL argument");
    static_assert(BP_TRACE_WORDS == 16, "ks_last_trace layout");
    CU_TRY(cudaSetDevice(s->device));
    unsigned long long tmp[BP_TRACE_WORDS];
    const cudaError_t e = bitpar_read_trace(s->bp, tmp);
    if (e == cudaErrorNotSupported) return fail(KS_ERR_INVALID, "no trace: run the process with KS_TRACE=1");
    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "trace read failed: %s", cudaGetErrorString(e));
    for (int k = 0; k < BP_TRACE_WORDS; k++) out_ns[k] = tmp[k];
    return KS_OK;
}

int ks_exchange_check(ks_snapshot* s) {
    if (!s) return fail(KS_ERR_INVALID, "snapshot is NULL");
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    CU_TRY(cudaDeviceSynchronize());
    int flag = 0;
    CU_TRY(cudaMemcpy(&flag, s->xflag.p, sizeof(int), cudaMemcpyDeviceToHost));
    if (flag) {
        CU_TRY(cudaMemset(s->xflag.p, 0, sizeof(int)));
        return fail(KS_ERR_CUDA, "exchange: a peer's bindings did not arrive within the timeout");
    }
    return KS_OK;
}

int ks_ipc_alloc(int device, uint64_t bytes, void** out_ptr, uint8_t out_handle[64]) {
    if (!out_ptr || !out_handle || bytes == 0) return fail(KS_ERR_INVALID, "bad ks_ipc_alloc argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    CU_TRY(cudaSetDevice(device));
    void* p = nullptr;
    CU_TRY(cudaMalloc(&p, bytes));
    cudaError_t e = cudaMemset(p, 0, bytes);
    cudaIpcMemHandle_t h;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        cudaFree(p);
        return fail(KS_ERR_CUDA, "ks_ipc_alloc failed: %s", cudaGetErrorString(e));
    }
    memcpy(out_handle, &h, 64);
    *out_ptr = p;
    return KS_OK;
}

int ks_ipc_open(int device, const uint8_t handle[64], void** out_ptr) {
    if (!out_ptr || !handle) return fail(KS_ERR_INVALID, "bad ks_ipc_open argument");
    CU_TRY(cudaSetDevice(device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    CU_TRY(cudaIpcOpenMemHandle(out_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return KS_OK;
}

int ks_ipc_close(int device, void* ptr) {
    if (!ptr) return KS_OK;
    CU_TRY(cudaSetDevice(device));
    CU_TRY(cudaIpcCloseMemHandle(ptr));
    return KS_OK;
}

int ks_measure_write_bandwidth(int device, void* dev_buf, uint64_t bytes, int iters, double* out_gbs) {
    if (!dev_buf || !out_gbs || bytes < (1u << 20) || ((uintptr_t)dev_buf & 31u)) return fail(KS_ERR_INVALID, "bad argument");
    CU_TRY(cudaSetDevice(device));
    int sms = 0;
    CU_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    Event e0, e1;
    CU_TRY(cudaEventCreate(&e0.h));
    CU_TRY(cudaEventCreate(&e1.h));
    float best = 1e30f;
    for (int it = 0; it < std::max(2, iters); it++) { // first pass untimed
        CU_TRY(cudaEventRecord(e0, nullptr));
        CU_TRY(launch_fill256(dev_buf, bytes, 0x5a5a0000u + (uint32_t)it, sms, nullptr));
        CU_TRY(cudaEventRecord(e1, nullptr));
        CU_TRY(cudaEventSynchronize(e1));
        float ms = 0;
        CU_TRY(cudaEventElapsedTime(&ms, e0, e1));
        if (it > 0) best = std::min(best, ms);
    }
    *out_gbs = (double)(bytes / 32 * 32) / (best * 1e-3) / 1e9;
    return KS_OK;
}

int ks_device_read(int device, const void* dev_ptr, void* host_ptr, uint64_t bytes) {
    if (!dev_ptr || !host_ptr) return fail(KS_ERR_INVALID, "NULL argument");
    CU_TRY(cudaSetDevice(device));
    CU_TRY(cudaDeviceSynchronize());
    CU_TRY(cudaMemcpy(host_ptr, dev_ptr, bytes, cudaMemcpyDeviceToHost));
    return KS_OK;
}

int ks_ipc_free(int device, void* ptr) {
    if (!ptr) return KS_OK;
    CU_TRY(cudaSetDevice(device));
    CU_TRY(cudaFree(ptr));
    return KS_OK;
}

int ks_snapshot_commit_claims(ks_snapshot* s, uint64_t n, const int32_t* claim_node, const int64_t* req_cpu,
                              const int64_t* req_mem, uint8_t* out_accepted) {
    if (!s) return fail(KS_ERR_INVALID, "snapshot is NULL");
    if (n && (!claim_node || !req_cpu || !req_mem || !out_accepted)) return fail(KS_ERR_INVALID, "NULL claim array");
    if (n == 0) return KS_OK;
    int rc = check_commit_requests(n, req_cpu, req_mem);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    s->derived_dirty = true;
    s->version++;
    const uint32_t chunk = stream_max_claims();
    CallerStaged plan;
    const auto node = plan.in(claim_node, n, 1, true);
    const auto cpu = plan.in(req_cpu, n, 1, true), mem = plan.in(req_mem, n, 1, true);
    const auto codes = plan.out(out_accepted, n, 1, true);
    CU_TRY(plan.reserve(s));
    CU_TRY(plan.upload(s->stream, 0, n));
    // chunks run in arrival order on one stream: per-node arrival order is preserved across chunks
    for (uint64_t off = 0; off < n; off += chunk) {
        const uint32_t m = (uint32_t)std::min<uint64_t>(chunk, n - off);
        CU_TRY(launch_stream_resolve(s->free_cpu.as<int64_t>(), s->free_mem.as<int64_t>(), plan.dev(node, off),
                                     plan.dev(cpu, off), plan.dev(mem, off), m, s->N, plan.dev(codes, off), s->stream));
    }
    CU_TRY(plan.download(s->stream, 0, n));
    CU_TRY(cudaStreamSynchronize(s->stream));
    return KS_OK;
}

int ks_select_sampling(ks_snapshot* s, const ks_pods* pods, uint32_t attempts, uint64_t seed, uint64_t first_pod_index,
                       int32_t* out_node_idx, uint32_t* out_attempts, int32_t* out_draw_node, uint8_t* out_draw_code) {
    int rc = check_pods(s, pods);
    if (rc) return rc;
    const uint64_t P = pods->n;
    if (P && !out_node_idx) return fail(KS_ERR_INVALID, "out_node_idx is NULL");
    if (attempts > 64) return fail(KS_ERR_RANGE, "attempts must be <= 64 (the reference uses %u)", KS_REFERENCE_ATTEMPTS);
    if (P == 0) return KS_OK;
    const uint64_t draws = P * (uint64_t)attempts;
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->N == 0 || attempts == 0) { // choose() on an empty store is None for every attempt (main.rs:56,60)
        for (uint64_t i = 0; i < P; i++) out_node_idx[i] = -1;
        if (out_attempts) memset(out_attempts, 0, P * 4);
        if (out_draw_node) memset(out_draw_node, 0xff, draws * 4);
        if (out_draw_code) memset(out_draw_code, 0xff, draws);
        return KS_OK;
    }
    CU_TRY(cudaSetDevice(s->device));
    CallerStaged plan;
    const StagedPods pd = declare_pods(plan, pods, s->W);
    const auto idx = plan.out(out_node_idx, P, 1, true);
    const auto used = plan.out(out_attempts, P, 1, true);
    const auto dn = plan.out(out_draw_node, P, attempts, true);
    const auto dc = plan.out(out_draw_code, P, attempts, true);
    CU_TRY(plan.reserve(s));
    CU_TRY(plan.upload(s->stream, 0, P));
    CU_TRY(launch_select_sampling(node_table(s), pd.view(plan, 0, P), attempts, seed, first_pod_index, plan.dev(idx),
                                  plan.dev(used), plan.dev(dn), plan.dev(dc), s->stream));
    CU_TRY(plan.download(s->stream, 0, P));
    CU_TRY(cudaStreamSynchronize(s->stream));
    return KS_OK;
}

int ks_explain(ks_snapshot* s, const ks_pods* pods, ks_pod_reasons* out, int32_t out_space, void* cuda_stream) {
    static_assert(sizeof(ks_pod_reasons) == 16, "ks_pod_reasons is four uint32");
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (!valid_space(out_space)) return fail(KS_ERR_INVALID, "bad out_space");
    const uint64_t P = pods->n;
    if (P && !out) return fail(KS_ERR_INVALID, "out is NULL");
    if (P == 0) return KS_OK;
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    const cudaStream_t st = call_stream(s, cuda_stream);
    CallerStaged plan;
    const StagedPods pd = declare_pods(plan, pods, s->W);
    const auto why = plan.out(reinterpret_cast<uint32_t*>(out), P, 4, out_space == KS_MEM_HOST);
    CU_TRY(plan.reserve(s));
    if (s->N == 0) {
        CU_TRY(plan.clear(st));
    } else {
        CU_TRY(plan.upload(st, 0, P));
        CU_TRY(launch_explain_counts(node_table(s), pd.view(plan, 0, P), plan.dev(why), s->sms, st));
    }
    CU_TRY(plan.download(st, 0, P));
    if (plan.any_host()) CU_TRY(cudaStreamSynchronize(st));
    return KS_OK;
}

int ks_select_topk(ks_snapshot* s, const ks_pods* pods, int policy, uint32_t k, int32_t* out_node_idx,
                   int64_t* out_score, uint32_t* out_feasible_cnt, int32_t out_space, void* cuda_stream) {
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (k == 0 || k > KS_TOPK_MAX) return fail(KS_ERR_RANGE, "k must be in [1, %u] (got %u)", KS_TOPK_MAX, k);
    if (!policy_valid(policy)) return fail(KS_ERR_INVALID, "bad policy");
    if (!valid_space(out_space)) return fail(KS_ERR_INVALID, "bad out_space");
    const uint64_t P = pods->n;
    if (P && !out_node_idx) return fail(KS_ERR_INVALID, "out_node_idx is NULL");
    if (P == 0) return KS_OK;
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    const cudaStream_t st = call_stream(s, cuda_stream);
    const bool host = out_space == KS_MEM_HOST;
    const DirectGrid g = s->N ? direct_grid(s->W, (uint32_t)P, s->Npad, s->sms) : DirectGrid{};
    const uint64_t part_rows = g.n_chunks > 1 ? (uint64_t)g.n_chunks * P : 0; // keys | indices | counts
    CallerStaged plan(&s->part_topk);
    const StagedPods pd = declare_pods(plan, pods, s->W);
    const auto idx = plan.out(out_node_idx, P, k, host, 0xff);
    const auto score = plan.out(out_score, P, k, host);
    const auto cnt = plan.out(out_feasible_cnt, P, 1, host);
    const auto pkey = plan.work<int64_t>(part_rows, k);
    const auto pidx = plan.work<int32_t>(part_rows, k);
    const auto pcnt = plan.work<uint32_t>(part_rows, 1);
    CU_TRY(plan.reserve(s));
    if (s->N == 0) { // no node: every slot is empty
        CU_TRY(plan.clear(st));
    } else {
        CU_TRY(plan.upload(st, 0, P));
        const OutView ov{plan.dev(idx), plan.dev(score), plan.dev(cnt), nullptr, 0, 0};
        const PartialView part{plan.dev(pkey), plan.dev(pidx), plan.dev(pcnt)};
        CU_TRY(launch_select_topk(node_table(s), pd.view(plan, 0, P), policy, k, ov, part, g, st));
    }
    CU_TRY(plan.download(st, 0, P));
    if (plan.any_host()) CU_TRY(cudaStreamSynchronize(st));
    return KS_OK;
}

// the bound list of ks_preempt against the snapshot's nodes: set_bound's checks plus the per-node sums of |request|
static int check_preempt_bound(const ks_snapshot* s, const ks_bound_pods* bound) {
    const uint64_t B = bound->n;
    std::vector<uint64_t> abs_sum;
    try {
        abs_sum.assign((size_t)s->N * 2, 0);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory checking %llu bound pods", (unsigned long long)B);
    }
    const uint64_t LIMIT = (uint64_t)KS_PREEMPT_MAX_ABS_SUM;
    for (uint64_t b = 0; b < B; b++) {
        const int32_t n = bound->node_idx[b];
        const int64_t c = bound->req_cpu[b], m = bound->req_mem[b];
        if (n < 0 || (uint32_t)n >= s->N)
            return fail(KS_ERR_INVALID, "bound pod %llu: node index %d out of range", (unsigned long long)b, n);
        if (!within_limits(c, m)) return fail(KS_ERR_RANGE, "bound pod %llu request out of range", (unsigned long long)b);
        uint64_t* a = &abs_sum[(size_t)n * 2];
        a[0] += (uint64_t)(c < 0 ? -c : c); // each term <= 2^55: no wrap before the sum passes the limit
        a[1] += (uint64_t)(m < 0 ? -m : m);
        if (a[0] > LIMIT || a[1] > LIMIT)
            return fail(KS_ERR_RANGE, "node %d: the bound pods' requests sum above 2^62 in absolute value", n);
    }
    return KS_OK;
}

int ks_preempt(ks_snapshot* s, const ks_pods* pods, const int32_t* pod_priority, const ks_bound_pods* bound,
               uint32_t max_victims, ks_preemption* out, int32_t* out_victims, int32_t out_space, void* cuda_stream) {
    static_assert(sizeof(ks_preemption) == 32, "ks_preemption is 32 bytes");
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (max_victims == 0 || max_victims > KS_PREEMPT_MAX_VICTIMS)
        return fail(KS_ERR_RANGE, "max_victims must be in [1, %u] (got %u)", KS_PREEMPT_MAX_VICTIMS, max_victims);
    if (!valid_space(out_space)) return fail(KS_ERR_INVALID, "bad out_space");
    const uint64_t P = pods->n;
    if (P && (!pod_priority || !out)) return fail(KS_ERR_INVALID, "pod_priority or out is NULL");
    if (!bound) return fail(KS_ERR_INVALID, "bound is NULL");
    const uint64_t B = bound->n;
    if (B && (!bound->node_idx || !bound->req_cpu || !bound->req_mem || !bound->priority))
        return fail(KS_ERR_INVALID, "NULL bound array");
    if (B > 0xffffffffull) return fail(KS_ERR_RANGE, "too many bound pods in one call");
    if (P == 0) return KS_OK;
    std::lock_guard<std::mutex> lk(s->mu);
    rc = check_preempt_bound(s, bound);
    if (rc) return rc;
    CU_TRY(cudaSetDevice(s->device));
    const cudaStream_t st = call_stream(s, cuda_stream);
    const bool host = out_space == KS_MEM_HOST;
    const DirectGrid g = s->N ? direct_grid(s->W, (uint32_t)P, s->Npad, s->sms) : DirectGrid{};
    const uint64_t part_rows = (uint64_t)g.n_chunks * P; // hi | lo | candidates | feasible
    CallerStaged plan(&s->part_pre);
    const StagedPods pd = declare_pods(plan, pods, s->W);
    const auto prio = plan.in(pod_priority, P, 1, pods->mem_space == KS_MEM_HOST);
    const auto rows = plan.out(out, P, 1, host);
    const auto vic = plan.out(out_victims, P, max_victims, host);
    const auto hi = plan.work<uint64_t>(part_rows, 1), lo = plan.work<uint64_t>(part_rows, 1);
    const auto cand = plan.work<uint32_t>(part_rows, 1), cnt = plan.work<uint32_t>(part_rows, 1);
    CU_TRY(plan.reserve(s));
    VictimIndex vx{};
    if (s->N) {
        CU_TRY(plan.upload(st, 0, P));
        // the victim index: upload the bound list, sort it by (node, priority), prefix sums per node
        CU_TRY(s->vx_pre.ensure(victim_index_bytes(B, s->N)));
        if (B) {
            const BoundUpload up = victim_index_inputs(s->vx_pre.p, B, s->N);
            CU_TRY(cudaMemcpyAsync(up.node, bound->node_idx, B * 4, cudaMemcpyHostToDevice, st));
            CU_TRY(cudaMemcpyAsync(up.cpu, bound->req_cpu, B * 8, cudaMemcpyHostToDevice, st));
            CU_TRY(cudaMemcpyAsync(up.mem, bound->req_mem, B * 8, cudaMemcpyHostToDevice, st));
            CU_TRY(cudaMemcpyAsync(up.prio, bound->priority, B * 4, cudaMemcpyHostToDevice, st));
        }
        CU_TRY(build_victim_index(s->vx_pre.p, B, s->N, &vx, st));
    }
    const PreemptPartials part{plan.dev(hi), plan.dev(lo), plan.dev(cand), plan.dev(cnt)};
    CU_TRY(launch_preempt(node_table(s), pd.view(plan, 0, P), plan.dev(prio), vx, max_victims, part, g, plan.dev(rows),
                          plan.dev(vic), st));
    CU_TRY(plan.download(st, 0, P));
    if (plan.any_host()) CU_TRY(cudaStreamSynchronize(st));
    return KS_OK;
}

int ks_stream_bind(ks_snapshot* s, const ks_pods* pods, int policy, int32_t* out_node_idx, int64_t* out_score,
                   uint32_t* out_rounds) {
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (pods->mem_space != KS_MEM_HOST) return fail(KS_ERR_INVALID, "ks_stream_bind takes host-space pods");
    if (pods->n && !out_node_idx) return fail(KS_ERR_INVALID, "out_node_idx is NULL");
    const uint64_t n = pods->n;
    const uint32_t W = s->W;
    if (!policy_valid(policy)) return fail(KS_ERR_INVALID, "bad policy");
    rc = check_commit_requests(n, pods->req_cpu, pods->req_mem);
    if (rc) return rc;
    if (n > 0 && n <= STREAM_BATCH_MAX && s->N > 0 && s->coop) {
        // device-side loop: the inputs [rc | rm | sel] and the results [score | idx | ctl] each travel as one block, so
        // the micro-batch costs ONE H2D copy, ONE cooperative launch that runs every round and ONE D2H copy
        std::lock_guard<std::mutex> lk(s->mu);
        CU_TRY(cudaSetDevice(s->device));
        HostStaged h;
        const auto cpu = h.in(pods->req_cpu, n), mem = h.in(pods->req_mem, n);
        const auto sel = h.in(pods->sel, n * W);
        const auto score = h.out(out_score, n);
        const auto idx = h.out(out_node_idx, n);
        const auto ctl = h.out<uint32_t>(nullptr, 2);
        const StreamBatchScratch w = stream_batch_scratch(h, s->sms);
        // sized for STREAM_BATCH_MAX pods on first use, so a stream of growing micro-batches never reallocates
        if (const int rc = h.reserve(s, (size_t)STREAM_BATCH_MAX * (16 + 8 * KS_MAX_LABEL_WORDS),
                                     (size_t)STREAM_BATCH_MAX * 12 + 8))
            return rc;
        cudaStream_t st = s->stream;
        CU_TRY(h.upload(st));
        StreamBatchArgs a = stream_batch_args(s, policy, h, w);
        a.m = (uint32_t)n;
        a.req_cpu = h.dev(cpu);
        a.req_mem = h.dev(mem);
        a.sel = h.dev(sel);
        a.ctl = h.dev(ctl);
        a.out_idx = h.dev(idx);
        a.out_score = h.dev(score);
        a.max_rounds = (uint32_t)n + 1;
        s->derived_dirty = true; // free[] changes: the bit-parallel index is stale
        s->version++;
        cudaError_t e = launch_stream_batch(a, W, st);
        if (e != cudaSuccess) return fail(KS_ERR_CUDA, "k_stream_batch launch failed: %s", cudaGetErrorString(e));
        CU_TRY(h.finish(st));
        if (out_rounds) *out_rounds = h.host(ctl)[1];
        s->last_path = "stream_batch";
        return KS_OK;
    }
    try { // host-driven loop (large batches, no cooperative launch): its vectors must not throw across the ABI
        std::vector<uint64_t> pending(n);
        for (uint64_t i = 0; i < n; i++) {
            pending[i] = i;
            out_node_idx[i] = -1;
            if (out_score) out_score[i] = 0;
        }
        std::vector<int64_t> rc_, rm_, score;
        std::vector<uint64_t> sel;
        std::vector<int32_t> idx;
        std::vector<uint8_t> acc;
        uint32_t rounds = 0;
        while (!pending.empty() && rounds <= n + 1) {
            const uint64_t m = pending.size();
            rc_.resize(m);
            rm_.resize(m);
            sel.resize(m * W);
            idx.resize(m);
            score.resize(m);
            acc.resize(m);
            for (uint64_t k = 0; k < m; k++) {
                const uint64_t p = pending[k];
                rc_[k] = pods->req_cpu[p];
                rm_[k] = pods->req_mem[p];
                for (uint32_t w = 0; w < W; w++) sel[k * W + w] = pods->sel[p * W + w];
            }
            ks_pods kp{m, rc_.data(), rm_.data(), sel.data(), KS_MEM_HOST};
            ks_bindings kb{idx.data(), score.data(), nullptr, KS_MEM_HOST, nullptr, 0, KS_MEM_HOST, nullptr, nullptr};
            rc = ks_select(s, &kp, policy, KS_SELECT_FORCE_DIRECT, &kb, nullptr); // claims against the current free[]
            if (rc) return rc;
            rc = ks_snapshot_commit_claims(s, m, idx.data(), rc_.data(), rm_.data(), acc.data());
            if (rc) return rc;
            std::vector<uint64_t> next;
            for (uint64_t k = 0; k < m; k++) {
                if (idx[k] < 0) continue; // no feasible node: NoNodeFound (src/main.rs:116-118)
                if (acc[k]) {
                    out_node_idx[pending[k]] = idx[k];
                    if (out_score) out_score[pending[k]] = score[k];
                } else {
                    next.push_back(pending[k]); // lost the node to an earlier pod of the batch: retry
                }
            }
            pending.swap(next);
            rounds++;
        }
        if (out_rounds) *out_rounds = rounds;
        return KS_OK;
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory in ks_stream_bind");
    }
}

// The cut of P pods into gangs->n groups of 1 to max_size pods each, and each min_member within its group's size
static int check_gangs(const ks_gangs* gangs, uint64_t P, uint64_t max_size) {
    const uint64_t G = gangs->n;
    const uint64_t* off = gangs->offset;
    if (off[0] != 0) return fail(KS_ERR_INVALID, "offset[0] must be 0");
    for (uint64_t g = 0; g < G; g++) {
        if (off[g + 1] < off[g]) return fail(KS_ERR_INVALID, "offsets decrease at group %llu", (unsigned long long)g);
        const uint64_t size = off[g + 1] - off[g];
        if (size == 0 || size > max_size)
            return fail(KS_ERR_RANGE, "group %llu has %llu pods (1..%llu)", (unsigned long long)g, (unsigned long long)size,
                        (unsigned long long)max_size);
        if (gangs->min_member[g] > size)
            return fail(KS_ERR_RANGE, "group %llu: min_member %u above its %llu pods", (unsigned long long)g,
                        gangs->min_member[g], (unsigned long long)size);
    }
    if (off[G] != P) return fail(KS_ERR_INVALID, "offset[n] must be pods->n");
    return KS_OK;
}

int ks_gang_bind(ks_snapshot* s, const ks_pods* pods, const ks_gangs* gangs, int policy, int32_t* out_node_idx,
                 int64_t* out_score, uint32_t* out_placed, uint32_t* out_rounds) {
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (pods->mem_space != KS_MEM_HOST) return fail(KS_ERR_INVALID, "ks_gang_bind takes host-space pods");
    if (!gangs || !gangs->offset || (gangs->n && !gangs->min_member)) return fail(KS_ERR_INVALID, "NULL group array");
    if (pods->n && !out_node_idx) return fail(KS_ERR_INVALID, "out_node_idx is NULL");
    if (!policy_valid(policy)) return fail(KS_ERR_INVALID, "bad policy");
    const uint64_t P = pods->n, G = gangs->n;
    const uint64_t* off = gangs->offset;
    rc = check_gangs(gangs, P, KS_GANG_MAX_SIZE);
    if (rc) return rc;
    if (G == 0) return KS_OK;
    rc = check_commit_requests(P, pods->req_cpu, pods->req_mem);
    if (rc) return rc;
    const uint32_t W = s->W;
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    if (!s->coop) return fail(KS_ERR_CUDA, "device %d has no cooperative launch", s->device);
    HostStaged h;
    const auto cpu = h.in(pods->req_cpu, P), mem = h.in(pods->req_mem, P);
    const auto sel = h.in(pods->sel, P * W);
    const auto offset = h.in<uint32_t>(nullptr, G + 1);
    const auto min_member = h.in(gangs->min_member, G);
    const auto score = h.out(out_score, P);
    const auto idx = h.out(out_node_idx, P);
    const auto ctl = h.out<uint32_t>(nullptr, 2 * G);
    const auto placed = h.out(out_placed, G);
    const StreamBatchScratch w = stream_batch_scratch(h, s->sms);
    if (const int rc = h.reserve(s)) return rc;
    for (uint64_t g = 0; g <= G; g++) h.host(offset)[g] = (uint32_t)off[g];
    cudaStream_t st = s->stream;
    CU_TRY(h.upload(st));
    StreamBatchArgs a = stream_batch_args(s, policy, h, w);
    a.m = (uint32_t)P;
    a.req_cpu = h.dev(cpu);
    a.req_mem = h.dev(mem);
    a.sel = h.dev(sel);
    a.ctl = nullptr; // per group: ga.ctl
    a.out_idx = h.dev(idx);
    a.out_score = h.dev(score);
    a.max_rounds = 0; // per group
    GangArgs ga;
    ga.n = (uint32_t)G;
    ga.offset = h.dev(offset);
    ga.min_member = h.dev(min_member);
    ga.ctl = h.dev(ctl);
    ga.placed = h.dev(placed);
    s->derived_dirty = true; // free[] changes: the bit-parallel index is stale
    s->version++;
    cudaError_t e = launch_gang_batch(a, ga, W, st);
    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "k_gang_batch launch failed: %s", cudaGetErrorString(e));
    CU_TRY(h.finish(st));
    if (out_rounds)
        for (uint64_t g = 0; g < G; g++) out_rounds[g] = h.host(ctl)[2 * g + 1];
    s->last_path = "gang_batch";
    return KS_OK;
}

// ks_drain_check's and ks_fit_drain_check's candidates: every check of ks_drain_check (include/ksched.h), in the order
// callers see them, then the round order - candidates by pod count descending, stable - and the candidates still
// running in each round.  Host code only; nothing is read from the device.
struct DrainPlan {
    uint64_t P = 0, D = 0;
    uint32_t rounds = 0;
    std::vector<uint32_t> order, per_round;
};

static int plan_drain(const ks_snapshot* s, const char* call, const ks_pods* pods, const ks_drain_candidates* cand,
                      int policy, uint32_t flags, const uint32_t* out_placed, const int32_t* out_node_idx, DrainPlan* pl) {
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (pods->mem_space != KS_MEM_HOST) return fail(KS_ERR_INVALID, "%s takes host-space pods", call);
    if (!cand || !cand->offset || (cand->n && (!cand->node_idx || !out_placed)))
        return fail(KS_ERR_INVALID, "NULL candidate array or out_placed");
    if (pods->n && !out_node_idx) return fail(KS_ERR_INVALID, "out_node_idx is NULL");
    if (!policy_valid(policy)) return fail(KS_ERR_INVALID, "bad policy");
    if (flags & ~KS_DRAIN_EXCLUDE_CANDIDATES) return fail(KS_ERR_INVALID, "unknown flags 0x%x", flags);
    const uint64_t P = pods->n, D = cand->n;
    const uint64_t* off = cand->offset;
    if (D > 0x7fffffffull) return fail(KS_ERR_RANGE, "too many candidates in one call");
    if (off[0] != 0) return fail(KS_ERR_INVALID, "offset[0] must be 0");
    uint32_t rounds = 0;
    for (uint64_t d = 0; d < D; d++) {
        if (off[d + 1] < off[d]) return fail(KS_ERR_INVALID, "offsets decrease at candidate %llu", (unsigned long long)d);
        const uint64_t size = off[d + 1] - off[d];
        if (size > KS_DRAIN_MAX_PODS)
            return fail(KS_ERR_RANGE, "candidate %llu has %llu pods (at most %u)", (unsigned long long)d,
                        (unsigned long long)size, KS_DRAIN_MAX_PODS);
        if (cand->node_idx[d] < 0 || (uint32_t)cand->node_idx[d] >= s->N)
            return fail(KS_ERR_INVALID, "candidate %llu: node index %d out of range", (unsigned long long)d,
                        cand->node_idx[d]);
        rounds = std::max(rounds, (uint32_t)size);
    }
    if (off[D] != P) return fail(KS_ERR_INVALID, "offset[n] must be pods->n");
    rc = check_commit_requests(P, pods->req_cpu, pods->req_mem); // P = 0 when D = 0
    if (rc) return rc;
    pl->P = P;
    pl->D = D;
    pl->rounds = rounds;
    std::vector<uint32_t>& order = pl->order; // candidates by pod count descending
    std::vector<uint32_t>& per_round = pl->per_round; // candidates still running in round r
    try {
        order.resize(D);
        per_round.assign(rounds, 0);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory ordering %llu candidates", (unsigned long long)D);
    }
    for (uint32_t d = 0; d < D; d++) order[d] = d;
    std::stable_sort(order.begin(), order.end(), [off](uint32_t a, uint32_t b) {
        return off[a + 1] - off[a] > off[b + 1] - off[b];
    });
    for (uint64_t d = 0; d < D; d++)
        for (uint64_t r = 0; r < off[d + 1] - off[d]; r++) per_round[r]++;
    return KS_OK;
}

int ks_drain_check(ks_snapshot* s, const ks_pods* pods, const ks_drain_candidates* cand, int policy, uint32_t flags,
                   uint32_t* out_placed, int32_t* out_node_idx, int64_t* out_score) {
    DrainPlan dp;
    const int rc = plan_drain(s, "ks_drain_check", pods, cand, policy, flags, out_placed, out_node_idx, &dp);
    if (rc || dp.D == 0) return rc;
    const uint64_t P = dp.P, D = dp.D;
    const uint64_t* off = cand->offset;
    const uint32_t rounds = dp.rounds;
    const std::vector<uint32_t>&order = dp.order, &per_round = dp.per_round;
    const uint32_t W = s->W;
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    // pods in round order, then the candidates in round order
    const bool excl = flags & KS_DRAIN_EXCLUDE_CANDIDATES;
    HostStaged h;
    const auto cpu = h.in<int64_t>(nullptr, P), mem = h.in<int64_t>(nullptr, P);
    const auto sel = h.in<uint64_t>(nullptr, P * W);
    const auto cand_node = h.in<int32_t>(nullptr, D);
    const auto pod_base = h.in<uint32_t>(nullptr, D), cand_id = h.in<uint32_t>(nullptr, D);
    const auto excluded = h.in<uint32_t>(nullptr, excl ? s->Npad / 32 : 0); // bits of the candidates' nodes
    const auto score = h.out(out_score, P);
    const auto idx = h.out(out_node_idx, P);
    const auto placed = h.out(out_placed, D);
    // node-chunk partials: the largest round needs the most
    uint64_t part_rows = 0;
    for (uint32_t r = 0; r < rounds; r++)
        part_rows = std::max<uint64_t>(part_rows, (uint64_t)direct_grid(W, per_round[r], s->Npad, s->sms).n_chunks * per_round[r]);
    const auto ov_fc = h.work<int64_t>(P), ov_fm = h.work<int64_t>(P), part_key = h.work<int64_t>(part_rows);
    const auto ov_node = h.work<int32_t>(P), part_idx = h.work<int32_t>(part_rows);
    const auto ov_cnt = h.work<uint32_t>(2 * D); // ov_cnt D, failed D: one array, zeroed together
    if (const int rc = h.reserve(s)) return rc;
    int64_t *h_rc = h.host(cpu), *h_rm = h.host(mem);
    uint64_t* h_sel = h.host(sel);
    int32_t* h_node = h.host(cand_node);
    uint32_t *h_base = h.host(pod_base), *h_id = h.host(cand_id);
    for (uint64_t j = 0; j < D; j++) {
        h_node[j] = cand->node_idx[order[j]];
        h_base[j] = (uint32_t)off[order[j]];
        h_id[j] = order[j];
    }
    for (uint64_t r = 0, r0 = 0; r < rounds; r0 += per_round[r], r++) // round r: pod r of the first per_round[r] candidates
        for (uint64_t j = 0; j < per_round[r]; j++) {
            const uint64_t p = off[order[j]] + r;
            h_rc[r0 + j] = pods->req_cpu[p];
            h_rm[r0 + j] = pods->req_mem[p];
            memcpy(h_sel + (r0 + j) * W, pods->sel + p * W, 8 * W);
        }
    if (excl) {
        uint32_t* h_excl = h.host(excluded);
        memset(h_excl, 0, excluded.n * 4);
        for (uint64_t d = 0; d < D; d++) h_excl[cand->node_idx[d] >> 5] |= 1u << (cand->node_idx[d] & 31);
    }
    cudaStream_t st = s->stream;
    CU_TRY(h.upload(st));
    CU_TRY(cudaMemsetAsync(h.dev(score), 0, P * 8, st));
    CU_TRY(cudaMemsetAsync(h.dev(idx), 0xff, P * 4, st));
    CU_TRY(cudaMemsetAsync(h.dev(placed), 0, D * 4, st));
    CU_TRY(cudaMemsetAsync(h.dev(ov_cnt), 0, D * 8, st));
    DrainArgs da;
    da.cand_node = h.dev(cand_node);
    da.pod_base = h.dev(pod_base);
    da.cand_id = h.dev(cand_id);
    da.excl = excl ? h.dev(excluded) : nullptr;
    da.ov_cnt = h.dev(ov_cnt);
    da.failed = da.ov_cnt + D;
    da.ov_node = h.dev(ov_node);
    da.ov_fc = h.dev(ov_fc);
    da.ov_fm = h.dev(ov_fm);
    da.out_idx = h.dev(idx);
    da.out_score = h.dev(score);
    da.placed = h.dev(placed);
    const PartialView part{h.dev(part_key), h.dev(part_idx), nullptr};
    const NodeTable nt = node_table(s);
    for (uint64_t r = 0, r0 = 0; r < rounds; r0 += per_round[r], r++) {
        const PodView pv{h.dev(cpu) + r0, h.dev(mem) + r0, h.dev(sel) + r0 * W, per_round[r]};
        const DirectGrid g = direct_grid(W, per_round[r], s->Npad, s->sms);
        cudaError_t e = launch_drain_round(nt, pv, da, policy, (uint32_t)r, part, g, st);
        if (e != cudaSuccess) return fail(KS_ERR_CUDA, "drain round %llu launch failed: %s", (unsigned long long)r, cudaGetErrorString(e));
    }
    CU_TRY(h.finish(st));
    s->last_path = "drain";
    return KS_OK;
}

// Every check of ks_scaleup_estimate (include/ksched.h), in the order callers see them; ks_fit_scaleup_estimate runs
// them first
static int check_scaleup(ks_snapshot* s, const char* call, const ks_pods* pods, const ks_node_templates* t,
                         const ks_scaleup_option* out, const int32_t* out_best) {
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (pods->mem_space != KS_MEM_HOST) return fail(KS_ERR_INVALID, "%s takes host-space pods", call);
    if (!t || !out_best) return fail(KS_ERR_INVALID, "NULL templates or out_best");
    const uint64_t P = pods->n, T = t->n;
    const uint32_t W = t->label_words;
    if (!valid_label_words(W)) return fail(KS_ERR_INVALID, "label_words must be 1, 2, 4 or 8 (got %u)", W);
    if (T && (!out || !t->alloc_cpu || !t->alloc_mem || !t->free_cpu || !t->free_mem || !t->labels || !t->max_nodes))
        return fail(KS_ERR_INVALID, "NULL template array or out");
    if (P > KS_SCALEUP_MAX_PODS) return fail(KS_ERR_RANGE, "%llu pods (at most %u)", (unsigned long long)P, KS_SCALEUP_MAX_PODS);
    if (T > KS_SCALEUP_MAX_TEMPLATES)
        return fail(KS_ERR_RANGE, "%llu templates (at most %u)", (unsigned long long)T, KS_SCALEUP_MAX_TEMPLATES);
    const int64_t lc = KS_MAX_CPU_MILLI >> 10, lm = KS_MAX_MEM_BYTES >> 10;
    for (uint64_t i = 0; i < T; i++) {
        const int64_t ac = t->alloc_cpu[i], am = t->alloc_mem[i], fc = t->free_cpu[i], fm = t->free_mem[i];
        if (ac < 1 || ac > lc || am < 1 || am > lm)
            return fail(KS_ERR_RANGE, "template %llu: allocatable (%lld millicores, %lld bytes) outside [1, 2^26] / [1, 2^45]",
                        (unsigned long long)i, (long long)ac, (long long)am);
        if (fc < -lc || fc > ac || fm < -lm || fm > am)
            return fail(KS_ERR_RANGE, "template %llu: capacity (%lld millicores, %lld bytes) outside [-2^26, allocatable] / "
                        "[-2^45, allocatable]", (unsigned long long)i, (long long)fc, (long long)fm);
        if (t->max_nodes[i] > KS_SCALEUP_MAX_NODES)
            return fail(KS_ERR_RANGE, "template %llu: max_nodes %u (at most %u)", (unsigned long long)i, t->max_nodes[i],
                        KS_SCALEUP_MAX_NODES);
    }
    return check_commit_requests(P, pods->req_cpu, pods->req_mem);
}

// The best template of the rows: most pods placed, then the highest utilization, then the fewest nodes, then the lowest
// index; -1 when none places a pod
static int32_t best_template(const ks_scaleup_option* out, uint64_t T) {
    int32_t best = -1;
    for (uint32_t i = 0; i < T; i++) {
        const ks_scaleup_option& r = out[i];
        if (r.placed == 0) continue;
        if (best < 0) {
            best = (int32_t)i;
            continue;
        }
        const ks_scaleup_option& b = out[best];
        if (r.placed > b.placed || (r.placed == b.placed && (r.utilization > b.utilization ||
                                                            (r.utilization == b.utilization && r.nodes < b.nodes))))
            best = (int32_t)i;
    }
    return best;
}

int ks_scaleup_estimate(ks_snapshot* s, const ks_pods* pods, const ks_node_templates* t, ks_scaleup_option* out,
                        int32_t* out_best, int32_t* out_node, ks_pod_reasons* out_reasons) {
    const int rc = check_scaleup(s, "ks_scaleup_estimate", pods, t, out, out_best);
    if (rc) return rc;
    const uint64_t P = pods->n, T = t->n;
    const uint32_t W = t->label_words;
    *out_best = -1;
    if (T == 0 || P == 0) { // nothing to pack: every row and reason count is zero
        if (T) memset(out, 0, T * sizeof(ks_scaleup_option));
        if (out_reasons && P) memset(out_reasons, 0, P * sizeof(ks_pod_reasons));
        return KS_OK;
    }
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    HostStaged h;
    const auto cpu = h.in(pods->req_cpu, P), mem = h.in(pods->req_mem, P), alloc_cpu = h.in(t->alloc_cpu, T),
               alloc_mem = h.in(t->alloc_mem, T), free_cpu = h.in(t->free_cpu, T), free_mem = h.in(t->free_mem, T);
    const auto sel = h.in(pods->sel, P * W), labels = h.in(t->labels, T * W);
    const auto max_nodes = h.in(t->max_nodes, T);
    const auto rows = h.out(out, T);
    const auto reasons = h.out(out_reasons, out_reasons ? P : 0, 16); // k_scaleup_reasons stores uint4
    const auto node = h.out(out_node, out_node ? T * P : 0);
    const uint32_t slots = scaleup_slots((uint32_t)T, s->sms);
    const auto scratch = h.work<uint32_t>((uint64_t)slots * 2 * P);
    if (const int rc = h.reserve(s)) return rc;
    cudaStream_t st = s->stream;
    CU_TRY(h.upload(st));
    if (out_node) CU_TRY(cudaMemsetAsync(h.dev(node), 0xff, T * P * 4, st));
    const PodView pv{h.dev(cpu), h.dev(mem), h.dev(sel), (uint32_t)P};
    ScaleupArgs a;
    a.T = (uint32_t)T;
    a.alloc_cpu = h.dev(alloc_cpu);
    a.alloc_mem = h.dev(alloc_mem);
    a.free_cpu = h.dev(free_cpu);
    a.free_mem = h.dev(free_mem);
    a.labels = h.dev(labels);
    a.max_nodes = h.dev(max_nodes);
    a.rows = h.dev(rows);
    a.out_node = out_node ? h.dev(node) : nullptr;
    a.reasons = out_reasons ? reinterpret_cast<uint32_t*>(h.dev(reasons)) : nullptr;
    a.scratch = h.dev(scratch);
    a.slots = slots;
    cudaError_t e = launch_scaleup(pv, W, a, st);
    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "scale-up launch failed: %s", cudaGetErrorString(e));
    CU_TRY(h.finish(st));
    *out_best = best_template(out, T);
    s->last_path = "scaleup";
    return KS_OK;
}

// The arguments ks_place_replicas and ks_place_replicas_spread share: host-space specs with requests that could be
// committed, a replica count per spec and the plan rows, a policy, and the limits on specs and copies.  *total = the
// copies asked for.
static int check_replica_specs(ks_snapshot* s, const char* call, const ks_pods* specs, const uint32_t* replicas,
                               const void* out, int policy, uint64_t* total) {
    int rc = check_pods(s, specs);
    if (rc) return rc;
    if (specs->mem_space != KS_MEM_HOST) return fail(KS_ERR_INVALID, "%s takes host-space specs", call);
    const uint64_t T = specs->n;
    if (T && (!replicas || !out)) return fail(KS_ERR_INVALID, "NULL replicas or out");
    if (!policy_valid(policy)) return fail(KS_ERR_INVALID, "bad policy");
    if (T > KS_REPLICAS_MAX_SPECS) return fail(KS_ERR_RANGE, "%llu specs (at most %u)", (unsigned long long)T, KS_REPLICAS_MAX_SPECS);
    *total = 0;
    for (uint64_t t = 0; t < T; t++) {
        if (replicas[t] > KS_REPLICAS_MAX)
            return fail(KS_ERR_RANGE, "spec %llu: %u replicas (at most %u)", (unsigned long long)t, replicas[t], KS_REPLICAS_MAX);
        *total += replicas[t];
    }
    if (*total > KS_REPLICAS_MAX_TOTAL)
        return fail(KS_ERR_RANGE, "%llu replicas in one call (at most %u)", (unsigned long long)*total, KS_REPLICAS_MAX_TOTAL);
    return check_commit_requests(T, specs->req_cpu, specs->req_mem);
}

int ks_place_replicas(ks_snapshot* s, const ks_pods* specs, const uint32_t* replicas, int policy, ks_replica_plan* out,
                      int32_t* out_node, int64_t* out_score) {
    uint64_t total;
    int rc = check_replica_specs(s, "ks_place_replicas", specs, replicas, out, policy, &total);
    if (rc) return rc;
    const uint64_t T = specs->n;
    if (T == 0) return KS_OK;
    const bool copies = out_node || out_score;
    if (s->N == 0) { // no node: nothing fits, every copy is -1
        memset(out, 0, T * sizeof(ks_replica_plan));
        if (out_node) memset(out_node, 0xff, total * 4);
        if (out_score) memset(out_score, 0, total * 8);
        return KS_OK;
    }
    const uint32_t W = s->W;
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    uint32_t n_chunks, chunk_len;
    replica_chunks(s->N, (uint32_t)T, s->sms, &n_chunks, &chunk_len);
    const uint64_t C = copies ? total : 0;
    uint32_t seq_ctas = 0, seq_block = 0;
    if (policy == KS_SCORE_LEAST_BALANCED) replica_seq_grid(s->N, (uint32_t)T, s->sms, &seq_ctas, &seq_block);
    HostStaged h;
    const auto cpu = h.in(specs->req_cpu, T), mem = h.in(specs->req_mem, T);
    const auto sel = h.in(specs->sel, T * W);
    const auto reps = h.in(replicas, T);
    const auto offset = h.in<uint64_t>(nullptr, T);
    const auto rows = h.out(out, T);
    const auto score = h.out(out_score, C);
    const auto node = h.out(out_node, C);
    const auto spec = h.work<unsigned char>(replica_spec_bytes((uint32_t)T), 16);
    const auto chunk = h.work<unsigned char>(replica_chunk_bytes((uint32_t)T, n_chunks), 16);
    const auto copy_score = h.work<int64_t>(C);
    const auto copy_node = h.work<int32_t>(C);
    const auto sort_buf = h.work<uint32_t>(2 * C);
    // KS_SCORE_LEAST_BALANCED: [scores | copies placed] per node and k_rep_seq CTA
    const auto seq_score = h.work<int64_t>((uint64_t)seq_ctas * s->N);
    const auto seq_placed = h.work<uint32_t>((uint64_t)seq_ctas * s->N);
    if (const int rc = h.reserve(s)) return rc;
    for (uint64_t t = 0, o = 0; t < T; o += replicas[t], t++) h.host(offset)[t] = o;
    cudaStream_t st = s->stream;
    CU_TRY(h.upload(st));
    if (copies) { // copies past `placed' stay -1 / 0
        CU_TRY(cudaMemsetAsync(h.dev(score), 0, C * 8, st));
        CU_TRY(cudaMemsetAsync(h.dev(node), 0xff, C * 4, st));
    }
    ReplicaArgs a;
    a.T = (uint32_t)T;
    a.req_cpu = h.dev(cpu);
    a.req_mem = h.dev(mem);
    a.sel = h.dev(sel);
    a.replicas = h.dev(reps);
    a.offset = h.dev(offset);
    a.rows = h.dev(rows);
    a.out_node = copies ? h.dev(node) : nullptr;
    a.out_score = copies ? h.dev(score) : nullptr;
    a.spec = reinterpret_cast<RepSpec*>(h.dev(spec));
    a.chunk = reinterpret_cast<RepChunk*>(h.dev(chunk));
    a.copy_node = copies ? h.dev(copy_node) : nullptr;
    a.copy_score = copies ? h.dev(copy_score) : nullptr;
    a.sort_buf = copies ? h.dev(sort_buf) : nullptr;
    a.n_chunks = n_chunks;
    a.chunk_len = chunk_len;
    ReplicaSeqArgs q;
    q.score = seq_ctas ? h.dev(seq_score) : nullptr;
    q.placed = seq_ctas ? h.dev(seq_placed) : nullptr;
    q.ctas = seq_ctas;
    q.block = seq_block;
    cudaError_t e = launch_replicas(node_table(s), policy, a, q, st);
    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "replica placement launch failed: %s", cudaGetErrorString(e));
    CU_TRY(h.finish(st));
    s->last_path = "replicas";
    return KS_OK;
}

// The keys of a ks_spread_multi against the snapshot's N nodes: 1 to KS_SPREAD_MAX_KEYS of them, each with a
// node_domain, 1 to KS_SPREAD_MAX_DOMAINS domains and every node's domain in [-1, D).  *S = the sum of the domains.
static int check_spread_keys(const ks_snapshot* s, const ks_spread_multi* spread, uint64_t* S) {
    const uint32_t NK = spread->n_keys, N = s->N;
    if (NK == 0 || NK > KS_SPREAD_MAX_KEYS) return fail(KS_ERR_RANGE, "%u topology keys (1 to %u)", NK, KS_SPREAD_MAX_KEYS);
    *S = 0;
    for (uint32_t k = 0; k < NK; k++) {
        if (!spread->node_domain[k]) return fail(KS_ERR_INVALID, "NULL spread, node_domain or max_skew");
        const uint32_t D = spread->n_domains[k];
        if (D == 0 || D > KS_SPREAD_MAX_DOMAINS) return fail(KS_ERR_RANGE, "%u domains (1 to %u)", D, KS_SPREAD_MAX_DOMAINS);
        for (uint32_t n = 0; n < N; n++)
            if (spread->node_domain[k][n] < -1 || spread->node_domain[k][n] >= (int64_t)D)
                return fail(KS_ERR_INVALID, "key %u, node %u: domain %d outside [-1, %u)", k, n, spread->node_domain[k][n], D);
        *S += D;
    }
    return KS_OK;
}

// ks_place_replicas_spread is the K = 1 case of ks_place_replicas_spread_multi: one argument check, one staging plan
// and one launcher for both.
static int place_spread(ks_snapshot* s, const char* call, const ks_pods* specs, const uint32_t* replicas,
                        const ks_spread_multi* spread, int policy, ks_spread_plan* out, int32_t* out_node,
                        int64_t* out_score, uint32_t* out_domain_count) {
    uint64_t total;
    int rc = check_replica_specs(s, call, specs, replicas, out, policy, &total);
    if (rc) return rc;
    const uint64_t T = specs->n;
    if (!spread || !spread->max_skew) return fail(KS_ERR_INVALID, "NULL spread, node_domain or max_skew");
    const uint32_t NK = spread->n_keys, N = s->N;
    uint64_t Stot;
    rc = check_spread_keys(s, spread, &Stot);
    if (rc) return rc;
    for (uint64_t i = 0; i < T * NK; i++)
        if (spread->max_skew[i] == 0)
            return fail(KS_ERR_RANGE, "spec %llu, key %llu: max_skew 0 (at least 1)", (unsigned long long)(i / NK),
                        (unsigned long long)(i % NK));
    const uint64_t TD = T * Stot;
    if ((spread->existing || out_domain_count) && TD > KS_SPREAD_MAX_COUNTS)
        return fail(KS_ERR_RANGE, "%llu specs x %llu domains of counts (at most 2^26)", (unsigned long long)T,
                    (unsigned long long)Stot);
    if (spread->existing)
        for (uint64_t i = 0; i < TD; i++)
            if (spread->existing[i] > KS_SPREAD_MAX_EXISTING)
                return fail(KS_ERR_RANGE, "spec %llu, count %llu: %u existing pods (at most 2^24)",
                            (unsigned long long)(i / Stot), (unsigned long long)(i % Stot), spread->existing[i]);
    if (T == 0) return KS_OK;
    const bool copies = out_node || out_score;
    if (N == 0) { // no node: no eligible domain, every copy is -1
        for (uint64_t t = 0; t < T * NK; t++) out[t] = ks_spread_plan{0, 0, 0, 0, 0, -1, 0};
        if (out_node) memset(out_node, 0xff, total * 4);
        if (out_score) memset(out_score, 0, total * 8);
        if (out_domain_count) {
            if (spread->existing) memcpy(out_domain_count, spread->existing, TD * 4);
            else memset(out_domain_count, 0, TD * 4);
        }
        return KS_OK;
    }
    // internal key order: the primary (fewest domains, then the lower key) first, the others in the caller's order
    uint32_t col[KS_SPREAD_MAX_KEYS] = {}, Dk[KS_SPREAD_MAX_KEYS] = {}, P[KS_SPREAD_MAX_KEYS] = {};
    for (uint32_t k = 0, p = 0; k < NK; p += spread->n_domains[k], k++) {
        P[k] = p;
        if (spread->n_domains[k] < spread->n_domains[col[0]]) col[0] = k;
    }
    for (uint32_t k = 0, i = 1; k < NK; k++)
        if (k != col[0]) col[i++] = k;
    for (uint32_t i = 0; i < NK; i++) Dk[i] = spread->n_domains[col[i]];
    const uint32_t W = s->W, D = Dk[0];
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    const uint64_t C = copies ? total : 0, E = spread->existing ? TD : 0, K = out_domain_count ? TD : 0;
    const uint64_t cta_bytes = spread_cta_bytes_keys(N, Dk, NK);
    uint32_t ctas;
    uint64_t seq_bytes;
    spread_seq_grid(cta_bytes, (uint32_t)T, s->sms, &ctas, &seq_bytes);
    HostStaged h;
    const auto cpu = h.in(specs->req_cpu, T), mem = h.in(specs->req_mem, T);
    const auto sel = h.in(specs->sel, T * W);
    const auto reps = h.in(replicas, T);
    const auto offset = h.in<uint64_t>(nullptr, T);
    const auto max_skew = h.in(spread->max_skew, T * NK);
    const auto min_domains = h.in(spread->min_domains, spread->min_domains ? T * NK : 0);
    Staged<int32_t> node_domain[KS_SPREAD_MAX_KEYS];
    for (uint32_t i = 0; i < NK; i++) node_domain[i] = h.in(spread->node_domain[col[i]], N);
    const auto existing = h.in(spread->existing, E);
    const auto rows = h.out(out, T * NK);
    const auto score = h.out(out_score, C);
    const auto node = h.out(out_node, C);
    const auto count = h.out(out_domain_count, K);
    Staged<uint32_t> sort_buf[KS_SPREAD_MAX_KEYS], perm[KS_SPREAD_MAX_KEYS], pos[KS_SPREAD_MAX_KEYS],
        dstart[KS_SPREAD_MAX_KEYS];
    for (uint32_t i = 0; i < NK; i++) {
        sort_buf[i] = h.work<uint32_t>(2ull * N);
        perm[i] = h.work<uint32_t>(N);
        pos[i] = h.work<uint32_t>(N);
        dstart[i] = h.work<uint32_t>((uint64_t)Dk[i] + 1);
    }
    const auto seq = h.work<unsigned char>(seq_bytes, 16); // k_spread_seq's scratch
    if (const int rc = h.reserve(s)) return rc;
    for (uint64_t t = 0, o = 0; t < T; o += replicas[t], t++) h.host(offset)[t] = o;
    cudaStream_t st = s->stream;
    CU_TRY(h.upload(st));
    if (copies) { // copies past `placed' stay -1 / 0
        CU_TRY(cudaMemsetAsync(h.dev(score), 0, C * 8, st));
        CU_TRY(cudaMemsetAsync(h.dev(node), 0xff, C * 4, st));
    }
    ReplicaArgs a{};
    a.T = (uint32_t)T;
    a.req_cpu = h.dev(cpu);
    a.req_mem = h.dev(mem);
    a.sel = h.dev(sel);
    a.replicas = h.dev(reps);
    a.offset = h.dev(offset);
    a.out_node = copies ? h.dev(node) : nullptr;
    a.out_score = copies ? h.dev(score) : nullptr;
    SpreadOrders o{};
    SpreadArgs q{};
    SpreadKeys mk{};
    o.K = mk.K = NK;
    for (uint32_t i = 0; i < NK; i++) {
        SpreadOrder& k = o.key[i];
        k.node_domain = h.dev(node_domain[i]);
        k.sort_buf = h.dev(sort_buf[i]);
        k.perm = h.dev(perm[i]);
        k.pos = h.dev(pos[i]);
        k.dstart = h.dev(dstart[i]);
        k.D = Dk[i];
        mk.col[i] = col[i];
        mk.off[i] = P[col[i]];
        mk.Dk[i] = Dk[i];
        mk.dom[i] = k.node_domain;
        mk.kperm[i] = k.perm;
        mk.kdstart[i] = k.dstart;
    }
    q.D = D;
    q.node_domain = o.key[0].node_domain;
    q.perm = o.key[0].perm;
    q.pos = o.key[0].pos;
    q.dstart = o.key[0].dstart;
    q.max_skew = h.dev(max_skew);
    q.min_domains = spread->min_domains ? h.dev(min_domains) : nullptr;
    q.existing = E ? h.dev(existing) : nullptr;
    q.rows = h.dev(rows);
    q.out_count = K ? h.dev(count) : nullptr;
    q.scratch = h.dev(seq);
    q.ctas = ctas;
    mk.S = (uint32_t)Stot;
    mk.cta_bytes = cta_bytes;
    cudaError_t e = launch_spread(node_table(s), policy, a, o, q, mk, st);
    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "spread placement launch failed: %s", cudaGetErrorString(e));
    CU_TRY(h.finish(st));
    s->last_path = "spread";
    return KS_OK;
}

int ks_place_replicas_spread(ks_snapshot* s, const ks_pods* specs, const uint32_t* replicas, const ks_spread* spread,
                             int policy, ks_spread_plan* out, int32_t* out_node, int64_t* out_score,
                             uint32_t* out_domain_count) {
    ks_spread_multi m{};
    if (spread) {
        m.n_keys = 1;
        m.n_domains[0] = spread->n_domains;
        m.node_domain[0] = spread->node_domain;
        m.max_skew = spread->max_skew;
        m.min_domains = spread->min_domains;
        m.existing = spread->existing;
    }
    return place_spread(s, "ks_place_replicas_spread", specs, replicas, spread ? &m : nullptr, policy, out, out_node,
                        out_score, out_domain_count);
}

int ks_place_replicas_spread_multi(ks_snapshot* s, const ks_pods* specs, const uint32_t* replicas,
                                   const ks_spread_multi* spread, int policy, ks_spread_plan* out, int32_t* out_node,
                                   int64_t* out_score, uint32_t* out_domain_count) {
    return place_spread(s, "ks_place_replicas_spread_multi", specs, replicas, spread, policy, out, out_node, out_score,
                        out_domain_count);
}

// ks_affinity_bind's terms compiled on the host (include/ksched.h, DESIGN.md 5n): the counter bases per (group, key),
// the first-pod flag per group and each group's deduplicated update entries.  With ks_profile_bind's scoring (5o), also
// the InterPodAffinity counters I_{g,k} and per bound group h the entries (g, k, c_{g,k}(h)) with c != 0.
struct AffinityPlan {
    std::vector<uint32_t> abase;   // [G * K * 2]: B_{g,k}, A_{g,k} bases, AFF_NONE = none
    std::vector<uint32_t> aflag;   // [G]
    std::vector<uint32_t> upd_off; // [G + 1]
    std::vector<uint32_t> upd;     // h | k << 16 | kind << 20
    uint64_t words = 0;            // counter words, the G first-pod words included
    uint32_t any_base = 0;
    std::vector<uint32_t> ibase;    // [G * K]: base of I_{g,k} (int64 words), AFF_NONE = none
    std::vector<uint32_t> iupd_off; // [G + 1]
    std::vector<uint32_t> iupd;     // g | k << 16
    std::vector<int32_t> icoef;     // c_{g,k}(h)
    uint64_t iwords = 0;
};

// c_{g,k}(h) of every (bound group h, incoming group g, key k), summed over the terms (include/ksched.h, 5o)
static int compile_scoring(const ks_pod_affinity* f, const ks_bind_scoring* sc, uint32_t G, uint32_t K,
                           const uint32_t* Dk, AffinityPlan* pl) {
    std::vector<std::pair<uint64_t, int64_t>> c; // (h << 32 | g << 4 | k, coefficient)
    std::vector<int32_t> tg;
    auto add = [&](uint32_t h, uint32_t g, uint32_t k, int64_t v) { c.emplace_back((uint64_t)h << 32 | g << 4 | k, v); };
    for (uint32_t t = 0; t < f->n_terms; t++) {
        const uint32_t o = (uint32_t)f->owner[t], k = f->key[t], kind = f->kind[t];
        const int64_t w = sc->term_weight ? sc->term_weight[t] : 0;
        if (kind == KS_POD_ANTI_AFFINITY || (kind == KS_POD_AFFINITY && sc->hard_affinity_weight == 0)) continue;
        tg.assign(f->target + f->target_offset[t], f->target + f->target_offset[t + 1]); // a term matches a pod once
        std::sort(tg.begin(), tg.end());
        tg.erase(std::unique(tg.begin(), tg.end()), tg.end());
        for (const int32_t h : tg) {
            if (kind == KS_POD_AFFINITY) { // an existing pod's required affinity term that matches the incoming pod
                add(o, (uint32_t)h, k, sc->hard_affinity_weight);
                continue;
            }
            const int64_t v = kind == KS_POD_AFFINITY_PREFERRED ? w : -w;
            add((uint32_t)h, o, k, v); // the incoming pod's term, against a bound pod of h
            add(o, (uint32_t)h, k, v); // the bound pod's term, against an incoming pod of h
        }
    }
    std::sort(c.begin(), c.end());
    std::vector<std::pair<uint64_t, int64_t>> m;
    for (const auto& e : c) {
        if (!m.empty() && m.back().first == e.first) m.back().second += e.second;
        else m.push_back(e);
    }
    m.erase(std::remove_if(m.begin(), m.end(), [](const auto& e) { return e.second == 0; }), m.end());
    if (m.size() > KS_AFFINITY_MAX_UPDATES)
        return fail(KS_ERR_RANGE, "%llu scoring update entries (at most 2^24)", (unsigned long long)m.size());
    pl->ibase.assign((size_t)G * K, AFF_NONE);
    pl->iupd_off.assign(G + 1, 0);
    pl->iupd.reserve(m.size());
    pl->icoef.reserve(m.size());
    for (const auto& e : m) {
        const uint32_t h = (uint32_t)(e.first >> 32), g = (uint32_t)(e.first >> 4 & 0xfffffffu), k = e.first & 15u;
        pl->iupd_off[h + 1]++;
        pl->iupd.push_back(g | k << 16);
        pl->icoef.push_back((int32_t)e.second); // |c| <= 2 * 100 * KS_AFFINITY_MAX_TERMS
        pl->ibase[(size_t)g * K + k] = 0;
    }
    for (uint32_t h = 0; h < G; h++) pl->iupd_off[h + 1] += pl->iupd_off[h];
    uint64_t word = 0;
    for (uint32_t g = 0; g < G; g++)
        for (uint32_t k = 0; k < K; k++)
            if (pl->ibase[(size_t)g * K + k] != AFF_NONE) {
                pl->ibase[(size_t)g * K + k] = (uint32_t)word;
                word += Dk[k];
                if (word > KS_SPREAD_MAX_COUNTS)
                    return fail(KS_ERR_RANGE, "more than 2^26 scoring counter words (group %u, key %u)", g, k);
            }
    pl->iwords = word;
    return KS_OK;
}

static int compile_affinity(const ks_pod_affinity* f, uint32_t G, uint32_t K, const uint32_t* Dk, uint32_t N,
                            AffinityPlan* pl, const ks_bind_scoring* sc = nullptr) {
    const uint32_t T = f->n_terms;
    const uint64_t E = f->n_existing;
    if (T > KS_AFFINITY_MAX_TERMS) return fail(KS_ERR_RANGE, "%u affinity terms (at most %u)", T, KS_AFFINITY_MAX_TERMS);
    if (E > KS_AFFINITY_MAX_EXISTING)
        return fail(KS_ERR_RANGE, "%llu existing pods (at most 2^24)", (unsigned long long)E);
    if (T && (!f->owner || !f->kind || !f->key || !f->target_offset))
        return fail(KS_ERR_INVALID, "NULL owner, kind, key or target_offset");
    if (E && (!f->existing_group || !f->existing_node)) return fail(KS_ERR_INVALID, "NULL existing_group or existing_node");
    for (uint32_t t = 0; t < T; t++) {
        if (f->owner[t] < 0 || f->owner[t] >= (int64_t)G)
            return fail(KS_ERR_INVALID, "term %u: owner %d outside [0, %u)", t, f->owner[t], G);
        if (!sc && f->kind[t] > KS_POD_ANTI_AFFINITY) return fail(KS_ERR_INVALID, "term %u: kind %u (0 or 1)", t, f->kind[t]);
        if (sc && f->kind[t] > KS_POD_ANTI_AFFINITY_PREFERRED)
            return fail(KS_ERR_INVALID, "term %u: kind %u (0 to 3)", t, f->kind[t]);
        const uint32_t w = sc && sc->term_weight ? sc->term_weight[t] : 0;
        if (sc && f->kind[t] >= KS_POD_AFFINITY_PREFERRED && (w < 1 || w > 100))
            return fail(KS_ERR_INVALID, "term %u: preferred term weight %u (1 to 100)", t, w);
        if (sc && f->kind[t] <= KS_POD_ANTI_AFFINITY && w)
            return fail(KS_ERR_INVALID, "term %u: required term weight %u (0)", t, w);
        if (f->key[t] >= K) return fail(KS_ERR_INVALID, "term %u: key %u (the call has %u)", t, f->key[t], K);
        if (f->target_offset[t + 1] < f->target_offset[t]) return fail(KS_ERR_INVALID, "term %u: target offsets decrease", t);
    }
    const uint64_t t0 = T ? f->target_offset[0] : 0, nt = T ? f->target_offset[T] - t0 : 0;
    if (nt > KS_AFFINITY_MAX_TARGETS) return fail(KS_ERR_RANGE, "%llu targets (at most 2^22)", (unsigned long long)nt);
    if (nt && !f->target) return fail(KS_ERR_INVALID, "NULL target");
    for (uint64_t i = t0; i < t0 + nt; i++)
        if (f->target[i] < 0 || f->target[i] >= (int64_t)G)
            return fail(KS_ERR_INVALID, "target %llu: group %d outside [0, %u)", (unsigned long long)i, f->target[i], G);
    for (uint64_t e = 0; e < E; e++) {
        if (f->existing_group[e] < 0 || f->existing_group[e] >= (int64_t)G)
            return fail(KS_ERR_INVALID, "existing pod %llu: group %d outside [0, %u)", (unsigned long long)e,
                        f->existing_group[e], G);
        if (f->existing_node[e] < 0 || f->existing_node[e] >= (int64_t)N)
            return fail(KS_ERR_INVALID, "existing pod %llu: node %d outside [0, %u)", (unsigned long long)e,
                        f->existing_node[e], N);
    }
    // anti[g * K + k]: B_{g,k} exists (an anti relation of g on k, in either direction); akeys[g]: g's affinity keys;
    // M[g]: the groups every affinity term of g targets, as a bitset of G bits
    const uint64_t words = (G + 63) / 64;
    std::vector<uint8_t> anti((size_t)G * K, 0), akeys(G, 0);
    std::vector<uint64_t> M((size_t)G * words, 0), tmp(words);
    std::vector<std::vector<uint32_t>> lists(G);
    auto enc = [](uint32_t g, uint32_t k, uint32_t kind) { return g | k << 16 | kind << 20; };
    for (uint32_t t = 0; t < T; t++) {
        const uint32_t g = (uint32_t)f->owner[t], k = f->key[t];
        if (f->kind[t] > KS_POD_ANTI_AFFINITY) continue; // preferred terms score only
        if (f->kind[t] == KS_POD_ANTI_AFFINITY) {
            anti[(size_t)g * K + k] = 1;
            for (uint64_t i = f->target_offset[t]; i < f->target_offset[t + 1]; i++) {
                const uint32_t h = (uint32_t)f->target[i];
                anti[(size_t)h * K + k] = 1;
                lists[h].push_back(enc(g, k, 0)); // rule 1: a pod of h raises g's count
                lists[g].push_back(enc(h, k, 0)); // rule 2: a pod of g (carrying the term) raises h's count
            }
            continue;
        }
        std::fill(tmp.begin(), tmp.end(), 0);
        for (uint64_t i = f->target_offset[t]; i < f->target_offset[t + 1]; i++)
            tmp[f->target[i] >> 6] |= 1ull << (f->target[i] & 63);
        uint64_t* m = M.data() + (size_t)g * words;
        for (uint64_t w = 0; w < words; w++) m[w] = akeys[g] ? m[w] & tmp[w] : tmp[w];
        akeys[g] |= (uint8_t)(1u << k);
    }
    // rule 3 adds |M_g| entries per affinity key of g, at most the targets of g's affinity terms: with rules 1 and 2's
    // two per anti target, every list together stays below 3 * KS_AFFINITY_MAX_TARGETS entries before deduplication
    pl->aflag.assign(G, 0);
    for (uint32_t g = 0; g < G; g++) {
        if (!akeys[g]) continue;
        const uint64_t* m = M.data() + (size_t)g * words;
        if (m[g >> 6] >> (g & 63) & 1) pl->aflag[g] = AFF_SELF;
        for (uint32_t h = 0; h < G; h++)
            if (m[h >> 6] >> (h & 63) & 1)
                for (uint32_t k = 0; k < K; k++)
                    if (akeys[g] >> k & 1) lists[h].push_back(enc(g, k, 1)); // rule 3: a pod of M_g raises A_{g,k}
    }
    pl->upd_off.assign(G + 1, 0);
    for (uint32_t h = 0; h < G; h++) {
        std::sort(lists[h].begin(), lists[h].end());
        lists[h].erase(std::unique(lists[h].begin(), lists[h].end()), lists[h].end());
        const uint64_t total = (uint64_t)pl->upd_off[h] + lists[h].size();
        if (total > KS_AFFINITY_MAX_UPDATES)
            return fail(KS_ERR_RANGE, "more than 2^24 update entries (%llu by group %u)", (unsigned long long)total, h);
        pl->upd_off[h + 1] = (uint32_t)total;
    }
    pl->upd.reserve(pl->upd_off[G]);
    for (uint32_t h = 0; h < G; h++) pl->upd.insert(pl->upd.end(), lists[h].begin(), lists[h].end());
    pl->abase.assign((size_t)G * K * 2, AFF_NONE);
    uint64_t word = 0;
    for (uint32_t g = 0; g < G; g++)
        for (uint32_t k = 0; k < K; k++) {
            if (anti[(size_t)g * K + k]) {
                pl->abase[((size_t)g * K + k) * 2] = (uint32_t)word;
                word += Dk[k];
            }
            if (akeys[g] >> k & 1) {
                pl->abase[((size_t)g * K + k) * 2 + 1] = (uint32_t)word;
                word += Dk[k];
            }
        }
    pl->any_base = (uint32_t)word;
    pl->words = word + G;
    if (pl->words > KS_SPREAD_MAX_COUNTS)
        return fail(KS_ERR_RANGE, "%llu affinity counter words (at most 2^26)", (unsigned long long)pl->words);
    return sc ? compile_scoring(f, sc, G, K, Dk, pl) : KS_OK;
}

// ks_node_bind's rules compiled on the host (include/ksched.h, DESIGN.md 5p): the class of each group (group -1 at 0),
// and per class its tolerations and its terms with their expressions, which point into the caller's expr_set
struct NodeRulesPlan {
    std::vector<uint32_t> cls;               // [G + 1]
    std::vector<uint64_t> ctol;              // [2C]: hard, soft
    std::vector<uint32_t> cterm_off{0};      // [C + 1]
    std::vector<uint32_t> cterm_w;           // [T']
    std::vector<uint32_t> cexpr_off{0};      // [T' + 1]
    std::vector<uint32_t> cexpr_key;         // [X']
    std::vector<uint64_t> cexpr_set;         // [X']: word offset of the set in expr_set
    uint64_t set_words = 0;                  // expr_set words the sets use
    uint32_t C = 0;
};

static int compile_node_rules(const ks_node_rules* r, uint32_t G, uint32_t N, NodeRulesPlan* pl) {
    if (r->weight_taint > 100 || r->weight_node_affinity > 100)
        return fail(KS_ERR_INVALID, "plugin weights %u and %u (at most 100)", r->weight_taint, r->weight_node_affinity);
    if (r->n_taints > KS_NODE_RULES_MAX_TAINTS) return fail(KS_ERR_RANGE, "%u taints (at most 64)", r->n_taints);
    if (r->n_keys > KS_NODE_RULES_MAX_KEYS)
        return fail(KS_ERR_RANGE, "%u node-affinity keys (at most %u)", r->n_keys, KS_NODE_RULES_MAX_KEYS);
    const uint64_t valid = r->n_taints == 64 ? ~0ull : (1ull << r->n_taints) - 1;
    const struct { const uint64_t* m; uint32_t n; const char* what; } masks[] = {
        {r->node_taint_hard, N, "node_taint_hard"}, {r->node_taint_soft, N, "node_taint_soft"},
        {r->tolerate_hard, G, "tolerate_hard"}, {r->tolerate_soft, G, "tolerate_soft"}};
    for (const auto& m : masks)
        if (m.m)
            for (uint32_t i = 0; i < m.n; i++)
                if (m.m[i] & ~valid) return fail(KS_ERR_INVALID, "%s[%u]: a taint bit at or above %u", m.what, i, r->n_taints);
    for (uint32_t k = 0; k < r->n_keys; k++) {
        if (N && !r->node_domain[k]) return fail(KS_ERR_INVALID, "NULL node_domain of node-affinity key %u", k);
        for (uint32_t n = 0; n < N; n++)
            if (r->node_domain[k][n] < -1 || r->node_domain[k][n] >= (int64_t)r->n_domains[k])
                return fail(KS_ERR_INVALID, "node-affinity key %u, node %u: domain %d outside [-1, %u)", k, n,
                            r->node_domain[k][n], r->n_domains[k]);
    }
    const uint32_t X = r->n_exprs, T = r->n_terms;
    if (X && (!r->expr_key || !r->expr_set_offset || !r->expr_set))
        return fail(KS_ERR_INVALID, "NULL expr_key, expr_set_offset or expr_set");
    if (T && (!r->term_owner || !r->term_weight || !r->term_expr_offset))
        return fail(KS_ERR_INVALID, "NULL term_owner, term_weight or term_expr_offset");
    for (uint32_t x = 0; x < X; x++) {
        const uint32_t k = r->expr_key[x];
        if (k >= r->n_keys) return fail(KS_ERR_INVALID, "expression %u: key %u (the call has %u)", x, k, r->n_keys);
        const uint64_t o = r->expr_set_offset[x], o1 = r->expr_set_offset[x + 1], D = r->n_domains[k];
        if (o1 < o || o1 - o != (D + 64) / 64)
            return fail(KS_ERR_INVALID, "expression %u: %llu set words (key %u needs %llu)", x,
                        (unsigned long long)(o1 < o ? 0 : o1 - o), k, (unsigned long long)((D + 64) / 64));
        if (o1 > KS_NODE_RULES_MAX_WORDS)
            return fail(KS_ERR_RANGE, "expression %u: set words beyond 2^26", x);
        const uint64_t top = r->expr_set[o1 - 1], used = (D + 1) % 64;
        if (used && (top >> used)) return fail(KS_ERR_INVALID, "expression %u: a set bit above D_k = %llu", x,
                                               (unsigned long long)D);
        pl->set_words = std::max(pl->set_words, o1);
    }
    std::vector<std::vector<uint32_t>> own(G);
    for (uint32_t t = 0; t < T; t++) {
        if (r->term_owner[t] < 0 || r->term_owner[t] >= (int64_t)G)
            return fail(KS_ERR_INVALID, "node-affinity term %u: owner %d outside [0, %u)", t, r->term_owner[t], G);
        if (r->term_weight[t] > 100) return fail(KS_ERR_INVALID, "node-affinity term %u: weight %u (0 to 100)", t,
                                                 r->term_weight[t]);
        if (r->term_expr_offset[t + 1] < r->term_expr_offset[t] || r->term_expr_offset[t + 1] > X)
            return fail(KS_ERR_INVALID, "node-affinity term %u: expression offsets decrease or pass %u", t, X);
        own[r->term_owner[t]].push_back(t);
    }
    for (uint32_t g = 0; g < G; g++) {
        uint32_t pref = 0;
        for (const uint32_t t : own[g]) pref += r->term_weight[t] != 0;
        if (pref > KS_NODE_RULES_MAX_PREFERRED)
            return fail(KS_ERR_RANGE, "group %u: %u preferred node-affinity terms (at most %u)", g, pref,
                        KS_NODE_RULES_MAX_PREFERRED);
    }
    // classes: the distinct signatures (tolerations, then each term's weight and expressions with their sets)
    std::map<std::vector<uint64_t>, uint32_t> seen;
    pl->cls.assign(G + 1, 0);
    auto add_class = [&](int64_t g) {
        std::vector<uint64_t> sig{g < 0 || !r->tolerate_hard ? 0 : r->tolerate_hard[g],
                                  g < 0 || !r->tolerate_soft ? 0 : r->tolerate_soft[g]};
        if (g >= 0)
            for (const uint32_t t : own[g]) {
                sig.push_back(r->term_weight[t]);
                sig.push_back(r->term_expr_offset[t + 1] - r->term_expr_offset[t]);
                for (uint32_t x = r->term_expr_offset[t]; x < r->term_expr_offset[t + 1]; x++) {
                    sig.push_back(r->expr_key[x]);
                    sig.insert(sig.end(), r->expr_set + r->expr_set_offset[x], r->expr_set + r->expr_set_offset[x + 1]);
                }
            }
        const auto it = seen.find(sig);
        if (it != seen.end()) return it->second;
        const uint32_t c = pl->C++;
        seen.emplace(std::move(sig), c);
        pl->ctol.push_back(g < 0 || !r->tolerate_hard ? 0 : r->tolerate_hard[g]);
        pl->ctol.push_back(g < 0 || !r->tolerate_soft ? 0 : r->tolerate_soft[g]);
        if (g >= 0)
            for (const uint32_t t : own[g]) {
                pl->cterm_w.push_back(r->term_weight[t]);
                for (uint32_t x = r->term_expr_offset[t]; x < r->term_expr_offset[t + 1]; x++) {
                    pl->cexpr_key.push_back(r->expr_key[x]);
                    pl->cexpr_set.push_back(r->expr_set_offset[x]);
                }
                pl->cexpr_off.push_back((uint32_t)pl->cexpr_key.size());
            }
        pl->cterm_off.push_back((uint32_t)pl->cterm_w.size());
        return c;
    };
    pl->cls[0] = add_class(-1);
    for (uint32_t g = 0; g < G; g++) pl->cls[g + 1] = add_class(g);
    if ((uint64_t)pl->C * N > KS_NODE_RULES_MAX_WORDS)
        return fail(KS_ERR_RANGE, "%u node-rule classes x %u nodes (at most 2^26 rule words)", pl->C, N);
    return KS_OK;
}

// ks_fit_bind's scalar resources (5r): at most KS_BIND_MAX_RESOURCES rows, every request at least 0
static int check_bind_resources(const ks_bind_resources* res, uint64_t P, uint32_t N) {
    const uint64_t RS = res->n_res;
    if (RS > KS_BIND_MAX_RESOURCES)
        return fail(KS_ERR_RANGE, "%llu resources (at most %u)", (unsigned long long)RS, KS_BIND_MAX_RESOURCES);
    if (RS && ((N && !res->node_free) || (P && !res->pod_req))) return fail(KS_ERR_INVALID, "NULL node_free or pod_req");
    for (uint64_t i = 0; i < P * RS; i++)
        if (res->pod_req[i] < 0)
            return fail(KS_ERR_RANGE, "pod %llu: request %lld of resource %llu (at least 0)", (unsigned long long)(i / RS),
                        (long long)res->pod_req[i], (unsigned long long)(i % RS));
    return KS_OK;
}

// last_path and the name in launch errors of each BindMode
static const char* const BIND_PATH[] = {"spread_bind", "affinity_bind", "profile_bind", "node_bind", "fit_bind",
                                        "gang_fit_bind"};
static const char* const BIND_NAME[] = {"spread bind", "affinity bind", "profile bind", "node bind", "fit bind",
                                        "gang fit bind"};

// One call of the bind walk, as its public entry (include/ksched.h) passes it.  Each mode reads what the mode before it
// reads and adds one part: AFFINITY aff (topo->max_skew may then be NULL), PROFILE scoring, NODE rules, FIT res and
// GANG_FIT gangs.  bind_spread reads a NULL aff, rules or res of the mode as empty; scoring and gangs are required.
struct BindOutputs {
    int32_t* node_idx = nullptr;      // [P], required
    int64_t* score = nullptr;         // [P]
    uint32_t* refused = nullptr;      // [P * bind_refusal_words(mode)]
    uint32_t* domain_count = nullptr; // [G * S]
    int64_t* parts = nullptr;         // [P * bind_part_words(mode)]
    uint32_t* soft_count = nullptr;   // [G * S]
    int64_t* free_r = nullptr;        // [R * N]
    uint32_t* placed = nullptr;       // [gangs->n]
};
struct BindRequest {
    const char* call = nullptr; // the public entry, in error messages
    BindMode mode = BIND_SPREAD;
    const ks_pods* pods = nullptr;
    const int32_t* group = nullptr;
    uint32_t n_groups = 0;
    const ks_spread_multi* topo = nullptr;
    int policy = 0;
    BindOutputs out{};
    const ks_pod_affinity* aff = nullptr;
    const ks_bind_scoring* scoring = nullptr;
    const ks_node_rules* rules = nullptr;
    const ks_bind_resources* res = nullptr;
    const ks_gangs* gangs = nullptr;
};

// What plan_bind derives from a request: the counts per group S, the walk's CTAs, first[g] = the first pod of group g or
// -1, the compiled terms and rules; and, filled by bind_spread once a walk runs, with scoring the domain bitmaps of the keys with more than one node in some
// domain (bit k of uniq: key k has none; bwo[k]: key k's word offset in each parity, BW words per parity).
struct BindPlan {
    uint64_t S = 0;
    uint32_t grid = 0;
    std::vector<int64_t> first;
    AffinityPlan aff;
    NodeRulesPlan rules;
    uint32_t uniq = 0, bwo[KS_SPREAD_MAX_KEYS] = {}, BW = 0;
};

// Every check of a bind call, in the order callers see them, then its plan; nothing has changed when it fails
static int plan_bind(const ks_snapshot* s, const BindRequest& r, BindPlan* pl) {
    const char* call = r.call;
    const ks_bind_scoring* sc = r.scoring;
    int rc = check_pods(s, r.pods);
    if (rc) return rc;
    if (r.pods->mem_space != KS_MEM_HOST) return fail(KS_ERR_INVALID, "%s takes host-space pods", call);
    if (!policy_valid(r.policy)) return fail(KS_ERR_INVALID, "bad policy");
    if (sc) {
        if (r.policy != KS_SCORE_LEAST_ALLOCATED && r.policy != KS_SCORE_MOST_ALLOCATED &&
            r.policy != KS_SCORE_LEAST_BALANCED)
            return fail(KS_ERR_INVALID, "%s takes policies 1, 3 and 4 (got %d)", call, r.policy);
        if (sc->hard_affinity_weight > 100 || sc->weight_spread > 100 || sc->weight_affinity > 100)
            return fail(KS_ERR_INVALID, "plugin weights %u, %u and hard affinity weight %u (at most 100)",
                        sc->weight_spread, sc->weight_affinity, sc->hard_affinity_weight);
        if (sc->soft_all_keys)
            for (uint32_t g = 0; g < r.n_groups; g++)
                if (sc->soft_all_keys[g] > 1)
                    return fail(KS_ERR_INVALID, "group %u: soft_all_keys %u (0 or 1)", g, sc->soft_all_keys[g]);
    }
    const ks_spread_multi* spread = r.topo;
    const uint64_t P = r.pods->n, G = r.n_groups;
    if (P && (!r.group || !r.out.node_idx)) return fail(KS_ERR_INVALID, "NULL group or out_node_idx");
    if (!spread || (G && !spread->max_skew && !r.aff)) return fail(KS_ERR_INVALID, "NULL spread, node_domain or max_skew");
    if (P > KS_SPREAD_BIND_MAX_PODS)
        return fail(KS_ERR_RANGE, "%llu pods (at most %u)", (unsigned long long)P, KS_SPREAD_BIND_MAX_PODS);
    if (G > KS_SPREAD_BIND_MAX_GROUPS)
        return fail(KS_ERR_RANGE, "%llu groups (at most %u)", (unsigned long long)G, KS_SPREAD_BIND_MAX_GROUPS);
    rc = check_spread_keys(s, spread, &pl->S);
    if (rc) return rc;
    const uint32_t K = spread->n_keys, W = s->W, N = s->N;
    const uint64_t S = pl->S, GS = G * S;
    if (GS > KS_SPREAD_MAX_COUNTS)
        return fail(KS_ERR_RANGE, "%llu groups x %llu domains of counts (at most 2^26)", (unsigned long long)G,
                    (unsigned long long)S);
    if (spread->existing)
        for (uint64_t i = 0; i < GS; i++)
            if (spread->existing[i] > KS_SPREAD_MAX_EXISTING)
                return fail(KS_ERR_RANGE, "group %llu, count %llu: %u existing pods (at most 2^24)",
                            (unsigned long long)(i / S), (unsigned long long)(i % S), spread->existing[i]);
    // every pod of a group carries the group's selector
    std::vector<int64_t>& first = pl->first;
    try {
        first.assign(G, -1);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory in %s", call);
    }
    for (uint64_t p = 0; p < P; p++) {
        const int32_t g = r.group[p];
        if (g < -1 || g >= (int64_t)G)
            return fail(KS_ERR_INVALID, "pod %llu: group %d outside [-1, %u)", (unsigned long long)p, g, r.n_groups);
        if (g < 0) continue;
        if (first[g] < 0) first[g] = (int64_t)p;
        else if (memcmp(r.pods->sel + p * W, r.pods->sel + first[g] * W, W * 8) != 0)
            return fail(KS_ERR_INVALID, "pod %llu: selector differs from pod %lld of group %d", (unsigned long long)p,
                        (long long)first[g], g);
    }
    rc = check_commit_requests(P, r.pods->req_cpu, r.pods->req_mem);
    if (!rc && r.res) rc = check_bind_resources(r.res, P, N);
    if (!rc && r.gangs && (!r.gangs->offset || (r.gangs->n && !r.gangs->min_member)))
        return fail(KS_ERR_INVALID, "NULL gang array");
    if (!rc && r.gangs) rc = check_gangs(r.gangs, P, KS_SPREAD_BIND_MAX_PODS); // a gang as large as the queue may be
    try {
        if (!rc && r.aff) rc = compile_affinity(r.aff, (uint32_t)G, K, spread->n_domains, N, &pl->aff, sc);
        if (!rc && r.rules) rc = compile_node_rules(r.rules, (uint32_t)G, N, &pl->rules);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory in %s", call);
    }
    pl->grid = std::max(1u, std::min<uint32_t>((uint32_t)s->sms, (N + 127u) / 128u));
    return rc;
}

// The staging of compiled node rules (NodeRulesPlan) for k_node_rules_setup, on a caller's HostStaged plan: the classes,
// the rule keys' domains, the taints and the sets, and one rule word per (class, node) in d_work.  With rules NULL every
// array is empty.  place() fills the arrays converted or defaulted in place and sets the NODE fields of ProfileBindArgs
// that k_node_rules_setup reads, and rules_grid; the caller sets q.b.N.
struct NodeRulesStage {
    HostStaged& h;
    const ks_node_rules* rules;
    const NodeRulesPlan& pl;
    const uint32_t N;
    const uint64_t NR = rules ? 1 : 0;
    Staged<uint32_t> ncls = h.in(pl.cls.data(), pl.cls.size());
    Staged<uint64_t> ctol = h.in(pl.ctol.data(), pl.ctol.size());
    Staged<uint32_t> cterm_off = h.in(pl.cterm_off.data(), NR * pl.cterm_off.size());
    Staged<uint32_t> cterm_w = h.in(pl.cterm_w.data(), pl.cterm_w.size());
    Staged<uint32_t> cexpr_off = h.in(pl.cexpr_off.data(), NR * pl.cexpr_off.size());
    Staged<uint32_t> cexpr_key = h.in(pl.cexpr_key.data(), pl.cexpr_key.size());
    Staged<uint64_t> cexpr_set = h.in(pl.cexpr_set.data(), pl.cexpr_set.size());
    Staged<uint64_t> nset = h.in(rules ? rules->expr_set : nullptr, pl.set_words);
    Staged<int32_t> ndom = h.in<int32_t>(nullptr, (uint64_t)(rules ? rules->n_keys : 0) * N);
    Staged<uint64_t> taint_hard = h.in(rules ? rules->node_taint_hard : nullptr, NR * N);
    Staged<uint64_t> taint_soft = h.in(rules ? rules->node_taint_soft : nullptr, NR * N);
    Staged<uint32_t> nrules = h.work<uint32_t>((uint64_t)pl.C * N);

    void place(ProfileBindArgs& q, int sms) const {
        const uint32_t KN = rules->n_keys;
        for (uint32_t k = 0; k < KN; k++) memcpy(h.host(ndom) + (size_t)k * N, rules->node_domain[k], (size_t)N * 4);
        if (!rules->node_taint_hard) memset(h.host(taint_hard), 0, (size_t)N * 8);
        if (!rules->node_taint_soft) memset(h.host(taint_soft), 0, (size_t)N * 8);
        q.ncls = h.dev(ncls);
        q.nrules = h.dev(nrules);
        q.C = pl.C;
        q.KN = KN;
        for (uint32_t k = 0; k < KN; k++) q.NDk[k] = rules->n_domains[k];
        q.ndom = h.dev(ndom);
        q.taint_hard = h.dev(taint_hard);
        q.taint_soft = h.dev(taint_soft);
        q.ctol = h.dev(ctol);
        q.cterm_off = h.dev(cterm_off);
        q.cterm_w = h.dev(cterm_w);
        q.cexpr_off = h.dev(cexpr_off);
        q.cexpr_key = h.dev(cexpr_key);
        q.cexpr_set = h.dev(cexpr_set);
        q.nset = h.dev(nset);
        q.rules_grid =
            (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(((uint64_t)q.C * N + 255) / 256, 4ull * (uint64_t)sms));
    }
};

// The staging of a bind call (ProfileBindArgs, ks_launch.h).  Building it declares every array on h in member order,
// feature by feature, with no element for a feature the mode does not read; after HostStaged::reserve(), place() fills
// the arrays converted or defaulted in place and points the kernel's fields at the staged arrays, in the same order.
// The compiled plans and the caller's host arrays are gathered from where they are.
struct BindStage {
    HostStaged& h;
    const ks_snapshot* s;
    const BindRequest& r;
    const BindPlan& pl;
    const uint64_t P = r.pods->n, G = r.n_groups, K = r.topo->n_keys, GS = G * pl.S, N = s->N, W = s->W;
    const uint64_t E = r.aff ? r.aff->n_existing : 0, Q = r.scoring ? 1 : 0, NR = r.rules ? 1 : 0;
    const uint64_t RS = r.res ? r.res->n_res : 0, NG = r.gangs ? r.gangs->n + 1 : 0, CTA = pl.grid;
    // every mode: the queue, the topology and the outputs
    Staged<int64_t> cpu = h.in(r.pods->req_cpu, P), mem = h.in(r.pods->req_mem, P);
    Staged<uint64_t> sel = h.in(r.pods->sel, P * W);
    Staged<int32_t> grp = h.in(r.group, P);
    Staged<uint32_t> max_skew = h.in(r.topo->max_skew, G * K);
    Staged<uint32_t> min_domains = h.in(r.topo->min_domains, r.topo->min_domains ? G * K : 0);
    Staged<uint32_t> existing = h.in(r.topo->existing, r.topo->existing ? GS : 0);
    Staged<int32_t> dom = h.in<int32_t>(nullptr, K * N);
    Staged<uint64_t> gsel = h.in<uint64_t>(nullptr, G * W);
    Staged<int64_t> score = h.out(r.out.score, P);
    Staged<int32_t> idx = h.out(r.out.node_idx, P);
    Staged<uint32_t> refused = h.out(r.out.refused, P * bind_refusal_words(r.mode));
    Staged<uint32_t> count = h.out(r.out.domain_count, GS); // the counts themselves: device state of the whole call
    Staged<uint8_t> elig = h.work<uint8_t>(GS);
    Staged<uint32_t> gk = h.work<uint32_t>(G * K * 4, 16);
    Staged<int64_t> pkey = h.work<int64_t>(CTA);
    Staged<int32_t> pidx = h.work<int32_t>(CTA);
    Staged<uint32_t> pref = h.work<uint32_t>(CTA);
    // AFFINITY on: the compiled terms, the existing pods and the counters
    Staged<uint32_t> abase = h.in(pl.aff.abase.data(), pl.aff.abase.size());
    Staged<uint32_t> aflag = h.in(pl.aff.aflag.data(), pl.aff.aflag.size());
    Staged<uint32_t> upd_off = h.in(pl.aff.upd_off.data(), pl.aff.upd_off.size());
    Staged<uint32_t> upd = h.in(pl.aff.upd.data(), pl.aff.upd.size());
    Staged<int32_t> ex_group = h.in(r.aff ? r.aff->existing_group : nullptr, E);
    Staged<int32_t> ex_node = h.in(r.aff ? r.aff->existing_node : nullptr, E);
    Staged<uint32_t> acnt = h.work<uint32_t>(pl.aff.words, 16);
    Staged<uint32_t> paref = h.work<uint32_t>(r.aff ? CTA : 0);
    // PROFILE on: the soft terms, the log table, the compiled IPA entries, the IPA counters and the domain bitmaps
    Staged<uint32_t> soft_skew = h.in(r.scoring ? r.scoring->soft_skew : nullptr, Q * G * K);
    Staged<uint8_t> soft_all = h.in(r.scoring ? r.scoring->soft_all_keys : nullptr, Q * G);
    Staged<double> logw = h.in<double>(nullptr, Q * (N + 2));
    Staged<uint32_t> ibase = h.in(pl.aff.ibase.data(), pl.aff.ibase.size());
    Staged<uint32_t> iupd_off = h.in(pl.aff.iupd_off.data(), pl.aff.iupd_off.size());
    Staged<uint32_t> iupd = h.in(pl.aff.iupd.data(), pl.aff.iupd.size());
    Staged<int32_t> icoef = h.in(pl.aff.icoef.data(), pl.aff.icoef.size());
    Staged<int64_t> parts = h.out(r.out.parts, Q * P * bind_part_words(r.mode));
    Staged<uint32_t> scnt = h.out(r.out.soft_count, Q * GS);
    Staged<int64_t> icnt = h.work<int64_t>(pl.aff.iwords, 16);
    Staged<uint32_t> bits = h.work<uint32_t>(2ull * pl.BW, 16);
    Staged<int64_t> iraw = h.work<int64_t>(Q * N), praw = h.work<int64_t>(Q * N);
    Staged<uint32_t> pdom = h.work<uint32_t>(Q * CTA * KS_SPREAD_MAX_KEYS), plack = h.work<uint32_t>(Q * CTA);
    Staged<int64_t> pimin = h.work<int64_t>(Q * CTA), pimax = h.work<int64_t>(Q * CTA);
    Staged<int64_t> ppmin = h.work<int64_t>(Q * CTA), ppmax = h.work<int64_t>(Q * CTA);
    // NODE on: the compiled classes and their rule words
    NodeRulesStage rs{h, r.rules, pl.rules, (uint32_t)N};
    Staged<uint32_t> ptref = h.work<uint32_t>(NR * CTA), pnref = h.work<uint32_t>(NR * CTA);
    Staged<uint32_t> ptmax = h.work<uint32_t>(NR * CTA), pnmax = h.work<uint32_t>(NR * CTA);
    // FIT on: the requests, the caller's free amounts and the charged ones, one row per resource
    Staged<int64_t> res_req = h.in(RS ? r.res->pod_req : nullptr, P * RS);
    Staged<int64_t> res_node_free = h.in(RS ? r.res->node_free : nullptr, RS * N);
    Staged<int64_t> res_free = h.out(r.out.free_r, RS * N);
    Staged<uint32_t> pfref = h.work<uint32_t>(r.res ? CTA : 0);
    // GANG_FIT: the gangs' offsets (NG of them) and minimums, their counts, and the rollback's group marks and lists
    Staged<uint32_t> goff = h.in<uint32_t>(nullptr, NG);
    Staged<uint32_t> gmin = h.in(r.gangs ? r.gangs->min_member : nullptr, r.gangs ? r.gangs->n : 0);
    Staged<uint32_t> gplaced = h.out(r.out.placed, r.gangs ? r.gangs->n : 0);
    Staged<uint32_t> gmark = h.work<uint32_t>(r.gangs ? 2 * G : 0), glist = h.work<uint32_t>(r.gangs ? 2 * G : 0);

    void place(ProfileBindArgs& q) const {
        const ks_spread_multi* t = r.topo;
        SpreadBindArgs& a = q.b;
        for (uint32_t k = 0; k < K; k++) memcpy(h.host(dom) + (size_t)k * N, t->node_domain[k], (size_t)N * 4);
        if (!t->max_skew) memset(h.host(max_skew), 0, G * K * 4); // AFFINITY on: zeros
        for (uint64_t g = 0; g < G; g++) {
            uint64_t* row = h.host(gsel) + g * W;
            if (pl.first[g] >= 0) memcpy(row, r.pods->sel + pl.first[g] * W, W * 8);
            else memset(row, 0, W * 8);
        }
        a.req_cpu = h.dev(cpu);
        a.req_mem = h.dev(mem);
        a.sel = h.dev(sel);
        a.group = h.dev(grp);
        a.gsel = h.dev(gsel);
        a.dom = h.dev(dom);
        a.max_skew = h.dev(max_skew);
        a.min_domains = t->min_domains ? h.dev(min_domains) : nullptr;
        a.existing = t->existing ? h.dev(existing) : nullptr;
        a.elig = h.dev(elig);
        a.gk = h.dev(gk);
        a.cnt = h.dev(count);
        a.pkey = h.dev(pkey);
        a.pidx = h.dev(pidx);
        a.pref = h.dev(pref);
        a.out_idx = h.dev(idx);
        a.out_score = h.dev(score);
        a.out_refused = h.dev(refused);
        if (r.aff) {
            a.abase = h.dev(abase);
            a.aflag = h.dev(aflag);
            a.upd_off = h.dev(upd_off);
            a.upd = h.dev(upd);
            a.ex_group = h.dev(ex_group);
            a.ex_node = h.dev(ex_node);
            a.E = (uint32_t)E;
            a.any_base = pl.aff.any_base;
            a.aff_grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((a.E + 7) / 8, 4ull * (uint64_t)s->sms));
            a.acnt = h.dev(acnt);
            a.paref = h.dev(paref);
        }
        if (const ks_bind_scoring* sc = r.scoring) {
            if (!sc->soft_skew) memset(h.host(soft_skew), 0, G * K * 4);
            if (!sc->soft_all_keys) memset(h.host(soft_all), 1, G);
            for (uint64_t i = 0; i < N + 2ull; i++) h.host(logw)[i] = log((double)(i + 2)); // the oracle's libm
            q.soft_skew = h.dev(soft_skew);
            q.soft_all = h.dev(soft_all);
            q.logw = h.dev(logw);
            q.uniq = pl.uniq;
            std::copy(pl.bwo, pl.bwo + K, q.bwo);
            q.BW = pl.BW;
            q.bits = h.dev(bits);
            q.scnt = h.dev(scnt);
            q.ibase = h.dev(ibase);
            q.iupd_off = h.dev(iupd_off);
            q.iupd = h.dev(iupd);
            q.icoef = h.dev(icoef);
            q.icnt = h.dev(icnt);
            q.iwords = pl.aff.iwords;
            q.iraw = h.dev(iraw);
            q.praw = h.dev(praw);
            q.pdom = h.dev(pdom);
            q.plack = h.dev(plack);
            q.pimin = h.dev(pimin);
            q.pimax = h.dev(pimax);
            q.ppmin = h.dev(ppmin);
            q.ppmax = h.dev(ppmax);
            q.out_parts = h.dev(parts);
            q.wspread = sc->weight_spread;
            q.waff = sc->weight_affinity;
        }
        if (const ks_node_rules* nr = r.rules) {
            rs.place(q, s->sms);
            q.ptref = h.dev(ptref);
            q.pnref = h.dev(pnref);
            q.ptmax = h.dev(ptmax);
            q.pnmax = h.dev(pnmax);
            q.wtaint = nr->weight_taint;
            q.wnaff = nr->weight_node_affinity;
        }
        if (r.res) {
            q.R = (uint32_t)RS;
            q.res_req = h.dev(res_req);
            q.res_node_free = h.dev(res_node_free);
            q.res_free = h.dev(res_free);
            q.pfref = h.dev(pfref);
        }
        if (const ks_gangs* gangs = r.gangs) {
            for (uint64_t j = 0; j <= gangs->n; j++) h.host(goff)[j] = (uint32_t)gangs->offset[j]; // P < 2^32
            q.n_gangs = (uint32_t)gangs->n;
            q.goff = h.dev(goff);
            q.gmin = h.dev(gmin);
            q.gplaced = h.dev(gplaced);
            q.gmark = h.dev(gmark);
            q.glist = h.dev(glist);
        }
    }
};

// The six bind entries' one call: plan_bind, the staging, one H2D copy, launch_bind and one D2H copy
static int bind_spread(ks_snapshot* s, const BindRequest& req) {
    static const ks_pod_affinity no_aff{};
    static const ks_node_rules no_rules{}; // no taint, no term, both plugin weights 0: the total is ks_profile_bind's
    static const ks_bind_resources no_res{};
    if (req.mode >= BIND_PROFILE && !req.scoring) return fail(KS_ERR_INVALID, "NULL scoring");
    if (req.mode == BIND_GANG_FIT && !req.gangs) return fail(KS_ERR_INVALID, "NULL gangs");
    BindRequest r = req;
    if (r.mode >= BIND_AFFINITY && !r.aff) r.aff = &no_aff;
    if (r.mode >= BIND_NODE && !r.rules) r.rules = &no_rules;
    if (r.mode >= BIND_FIT && !r.res) r.res = &no_res;
    BindPlan pl;
    const int rc = plan_bind(s, r, &pl);
    if (rc) return rc;
    const BindOutputs& o = r.out;
    const uint64_t P = r.pods->n, GS = (uint64_t)r.n_groups * pl.S, RS = r.res ? r.res->n_res : 0;
    const uint32_t N = s->N;
    if (o.free_r && RS && N && (P == 0)) memcpy(o.free_r, r.res->node_free, RS * N * 8); // nothing binds: L3
    if (o.placed) memset(o.placed, 0, r.gangs->n * 4); // rewritten by the walk when it runs
    if (P == 0) return KS_OK;
    if (N == 0) { // no node: nothing is placed, every count is existing
        memset(o.node_idx, 0xff, P * 4);
        if (o.score) memset(o.score, 0, P * 8);
        if (o.refused) memset(o.refused, 0, P * bind_refusal_words(r.mode) * 4);
        for (uint32_t* c : {o.domain_count, o.soft_count})
            if (c) {
                if (r.topo->existing) memcpy(c, r.topo->existing, GS * 4);
                else memset(c, 0, GS * 4);
            }
        if (o.parts) memset(o.parts, 0, P * bind_part_words(r.mode) * 8);
        return KS_OK;
    }
    for (uint32_t k = 0; r.scoring && k < r.topo->n_keys; k++) { // the domain bitmaps, once a walk runs
        const uint32_t D = r.topo->n_domains[k];
        std::vector<uint8_t> seen;
        try {
            seen.assign(D, 0);
        } catch (...) {
            return fail(KS_ERR_NOMEM, "out of host memory in %s", r.call);
        }
        bool uniq = true;
        for (uint32_t n = 0; n < N && uniq; n++) {
            const int32_t d = r.topo->node_domain[k][n];
            if (d >= 0) uniq = !seen[d]++;
        }
        pl.bwo[k] = pl.BW;
        if (uniq) pl.uniq |= 1u << k;
        else pl.BW += (D + 31) / 32;
    }
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    if (!s->coop) return fail(KS_ERR_CUDA, "device %d has no cooperative launch", s->device);
    ProfileBindArgs q{}; // the fields a mode does not read stay zero
    SpreadBindArgs& a = q.b;
    a.N = N;
    a.Npad = s->Npad;
    a.P = (uint32_t)P;
    a.G = r.n_groups;
    a.K = r.topo->n_keys;
    a.S = (uint32_t)pl.S;
    for (uint32_t k = 0, o = 0; k < a.K; o += r.topo->n_domains[k], k++) {
        a.Dk[k] = r.topo->n_domains[k];
        a.Pk[k] = o;
    }
    a.alloc_cpu = s->alloc_cpu.as<int64_t>();
    a.alloc_mem = s->alloc_mem.as<int64_t>();
    a.labels = s->labels.as<uint64_t>();
    a.free_cpu = s->free_cpu.as<int64_t>();
    a.free_mem = s->free_mem.as<int64_t>();
    a.policy = r.policy;
    a.grid = pl.grid;
    a.setup_grid = bind_setup_grid(r.n_groups, s->sms);
    HostStaged h;
    const BindStage stage{h, s, r, pl};
    if (const int e = h.reserve(s)) return e;
    stage.place(q);
    cudaStream_t st = s->stream;
    CU_TRY(h.upload(st));
    s->derived_dirty = true; // free[] changes: the bit-parallel index is stale
    s->version++;
    const cudaError_t e = launch_bind(r.mode, q, pl.aff.words, s->W, st);
    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "%s launch failed: %s", BIND_NAME[r.mode], cudaGetErrorString(e));
    CU_TRY(h.finish(st));
    s->last_path = BIND_PATH[r.mode];
    return KS_OK;
}

// ks_fit_bind and ks_gang_fit_bind: with rules NULL, parts words 3-4 read 0, as ks_node_bind's K1 gives them (M1)
static int bind_fit(ks_snapshot* s, const BindRequest& r) {
    const int rc = bind_spread(s, r);
    if (rc || r.rules || !r.out.parts) return rc;
    for (uint64_t p = 0; p < r.pods->n; p++) r.out.parts[5 * p + 3] = r.out.parts[5 * p + 4] = 0;
    return KS_OK;
}

int ks_spread_bind(ks_snapshot* s, const ks_pods* pods, const int32_t* group, uint32_t n_groups,
                   const ks_spread_multi* spread, int policy, int32_t* out_node_idx, int64_t* out_score,
                   uint32_t* out_refused, uint32_t* out_domain_count) {
    return bind_spread(s, {"ks_spread_bind", BIND_SPREAD, pods, group, n_groups, spread, policy,
                           {out_node_idx, out_score, out_refused, out_domain_count}});
}

int ks_affinity_bind(ks_snapshot* s, const ks_pods* pods, const int32_t* group, uint32_t n_groups,
                     const ks_spread_multi* topo, const ks_pod_affinity* aff, int policy, int32_t* out_node_idx,
                     int64_t* out_score, uint32_t* out_refused, uint32_t* out_domain_count) {
    return bind_spread(s, {"ks_affinity_bind", BIND_AFFINITY, pods, group, n_groups, topo, policy,
                           {out_node_idx, out_score, out_refused, out_domain_count}, aff});
}

int ks_profile_bind(ks_snapshot* s, const ks_pods* pods, const int32_t* group, uint32_t n_groups,
                    const ks_spread_multi* topo, const ks_pod_affinity* aff, const ks_bind_scoring* scoring, int policy,
                    int32_t* out_node_idx, int64_t* out_score, int64_t* out_parts, uint32_t* out_refused,
                    uint32_t* out_domain_count, uint32_t* out_soft_count) {
    return bind_spread(s, {"ks_profile_bind", BIND_PROFILE, pods, group, n_groups, topo, policy,
                           {out_node_idx, out_score, out_refused, out_domain_count, out_parts, out_soft_count}, aff,
                           scoring});
}

int ks_node_bind(ks_snapshot* s, const ks_pods* pods, const int32_t* group, uint32_t n_groups,
                 const ks_spread_multi* topo, const ks_pod_affinity* aff, const ks_bind_scoring* scoring,
                 const ks_node_rules* rules, int policy, int32_t* out_node_idx, int64_t* out_score, int64_t* out_parts,
                 uint32_t* out_refused, uint32_t* out_domain_count, uint32_t* out_soft_count) {
    BindRequest r{"ks_node_bind", BIND_NODE, pods, group, n_groups, topo, policy,
                  {out_node_idx, out_score, out_refused, out_domain_count, out_parts, out_soft_count}, aff, scoring,
                  rules};
    if (rules) return bind_spread(s, r);
    // K1: no rules is ks_profile_bind itself, its refusals and parts widened with zeros
    if (!scoring) return fail(KS_ERR_INVALID, "NULL scoring");
    const uint64_t P = pods ? pods->n : 0;
    std::vector<uint32_t> ref;
    std::vector<int64_t> parts;
    try {
        if (out_refused) ref.resize(2 * P);
        if (out_parts) parts.resize(3 * P);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory in ks_node_bind");
    }
    r.mode = BIND_PROFILE;
    r.out.refused = out_refused ? ref.data() : nullptr;
    r.out.parts = out_parts ? parts.data() : nullptr;
    const int rc = bind_spread(s, r);
    if (rc) return rc;
    for (uint64_t p = 0; p < P; p++) {
        if (out_refused) {
            out_refused[4 * p] = out_refused[4 * p + 1] = 0;
            out_refused[4 * p + 2] = ref[2 * p];
            out_refused[4 * p + 3] = ref[2 * p + 1];
        }
        if (out_parts) {
            for (int i = 0; i < 3; i++) out_parts[5 * p + i] = parts[3 * p + i];
            out_parts[5 * p + 3] = out_parts[5 * p + 4] = 0;
        }
    }
    return KS_OK;
}

int ks_fit_bind(ks_snapshot* s, const ks_pods* pods, const int32_t* group, uint32_t n_groups,
                const ks_spread_multi* topo, const ks_pod_affinity* aff, const ks_bind_scoring* scoring,
                const ks_node_rules* rules, const ks_bind_resources* res, int policy, int32_t* out_node_idx,
                int64_t* out_score, int64_t* out_parts, uint32_t* out_refused, uint32_t* out_domain_count,
                uint32_t* out_soft_count, int64_t* out_free) {
    return bind_fit(s, {"ks_fit_bind", BIND_FIT, pods, group, n_groups, topo, policy,
                        {out_node_idx, out_score, out_refused, out_domain_count, out_parts, out_soft_count, out_free},
                        aff, scoring, rules, res});
}

int ks_gang_fit_bind(ks_snapshot* s, const ks_pods* pods, const int32_t* group, uint32_t n_groups,
                     const ks_spread_multi* topo, const ks_pod_affinity* aff, const ks_bind_scoring* scoring,
                     const ks_node_rules* rules, const ks_bind_resources* res, const ks_gangs* gangs, int policy,
                     int32_t* out_node_idx, int64_t* out_score, int64_t* out_parts, uint32_t* out_refused,
                     uint32_t* out_domain_count, uint32_t* out_soft_count, int64_t* out_free, uint32_t* out_placed) {
    return bind_fit(s, {"ks_gang_fit_bind", BIND_GANG_FIT, pods, group, n_groups, topo, policy,
                        {out_node_idx, out_score, out_refused, out_domain_count, out_parts, out_soft_count, out_free,
                         out_placed},
                        aff, scoring, rules, res, gangs});
}

// ks_fit_preempt's bound requests against node_free (include/ksched.h): each >= 0, and per (r, n) |node_free| plus the
// sum over n's bound pods at most 2^62
static int check_fit_preempt_bound(const ks_snapshot* s, const ks_bound_pods* bound, const int64_t* bound_req,
                                   const ks_bind_resources* res) {
    const uint64_t B = bound->n, R = res->n_res, N = s->N;
    std::vector<uint64_t> sum;
    try {
        sum.assign(R * N, 0);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory checking %llu bound pods", (unsigned long long)B);
    }
    const uint64_t LIMIT = (uint64_t)KS_PREEMPT_MAX_ABS_SUM;
    for (uint64_t i = 0; i < R * N; i++) {
        const int64_t f = res->node_free[i];
        sum[i] = f < 0 ? 0 - (uint64_t)f : (uint64_t)f;
        if (sum[i] > LIMIT)
            return fail(KS_ERR_RANGE, "resource %llu, node %llu: |node_free| above 2^62", (unsigned long long)(i / N),
                        (unsigned long long)(i % N));
    }
    for (uint64_t b = 0; b < B; b++)
        for (uint64_t r = 0; r < R; r++) {
            const int64_t q = bound_req[b * R + r];
            if (q < 0)
                return fail(KS_ERR_RANGE, "bound pod %llu: request %lld of resource %llu (at least 0)",
                            (unsigned long long)b, (long long)q, (unsigned long long)r);
            uint64_t& a = sum[r * N + (uint32_t)bound->node_idx[b]]; // node range checked by check_preempt_bound
            if ((uint64_t)q > LIMIT - a)
                return fail(KS_ERR_RANGE, "resource %llu, node %d: |node_free| and the bound requests sum above 2^62",
                            (unsigned long long)r, bound->node_idx[b]);
            a += (uint64_t)q;
        }
    return KS_OK;
}

int ks_fit_preempt(ks_snapshot* s, const ks_pods* pods, const int32_t* group, uint32_t n_groups,
                   const ks_node_rules* rules, const ks_bind_resources* res, const int32_t* pod_priority,
                   const ks_bound_pods* bound, const int64_t* bound_req, uint32_t max_victims, ks_preemption* out,
                   int32_t* out_victims, uint32_t* out_unresolvable) {
    static const ks_node_rules no_rules{};
    static const ks_bind_resources no_res{};
    int rc = check_pods(s, pods);
    if (rc) return rc;
    if (pods->mem_space != KS_MEM_HOST) return fail(KS_ERR_INVALID, "ks_fit_preempt takes host-space pods");
    if (max_victims == 0 || max_victims > KS_PREEMPT_MAX_VICTIMS)
        return fail(KS_ERR_RANGE, "max_victims must be in [1, %u] (got %u)", KS_PREEMPT_MAX_VICTIMS, max_victims);
    const uint64_t P = pods->n, G = n_groups;
    if (P && (!pod_priority || !out)) return fail(KS_ERR_INVALID, "pod_priority or out is NULL");
    if (!bound) return fail(KS_ERR_INVALID, "bound is NULL");
    const uint64_t B = bound->n;
    if (B && (!bound->node_idx || !bound->req_cpu || !bound->req_mem || !bound->priority))
        return fail(KS_ERR_INVALID, "NULL bound array");
    if (B > 0xffffffffull) return fail(KS_ERR_RANGE, "too many bound pods in one call");
    if (P && !group) return fail(KS_ERR_INVALID, "NULL group");
    if (G > KS_SPREAD_BIND_MAX_GROUPS)
        return fail(KS_ERR_RANGE, "%llu groups (at most %u)", (unsigned long long)G, KS_SPREAD_BIND_MAX_GROUPS);
    for (uint64_t p = 0; p < P; p++)
        if (group[p] < -1 || group[p] >= (int64_t)G)
            return fail(KS_ERR_INVALID, "pod %llu: group %d outside [-1, %u)", (unsigned long long)p, group[p], n_groups);
    const ks_node_rules* nr = rules ? rules : &no_rules;
    if (!res) res = &no_res;
    const uint32_t N = s->N, R = res->n_res;
    rc = check_bind_resources(res, P, N);
    if (rc) return rc;
    if (R && B && !bound_req) return fail(KS_ERR_INVALID, "NULL bound_req");
    NodeRulesPlan rp;
    try {
        rc = compile_node_rules(nr, (uint32_t)G, N, &rp);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory in ks_fit_preempt");
    }
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(s->mu);
    rc = check_preempt_bound(s, bound);
    if (!rc) rc = check_fit_preempt_bound(s, bound, bound_req, res);
    if (rc || P == 0) return rc;
    CU_TRY(cudaSetDevice(s->device));
    const cudaStream_t st = s->stream;
    const DirectGrid g = N ? fit_preempt_grid((uint32_t)P, s->Npad, s->sms) : DirectGrid{};
    const uint64_t part_rows = (uint64_t)g.n_chunks * P;
    const size_t vx_bytes = N ? victim_index_bytes(B, N) : 0;
    HostStaged h;
    const Staged<int64_t> cpu = h.in(pods->req_cpu, P), mem = h.in(pods->req_mem, P);
    const Staged<uint64_t> sel = h.in(pods->sel, P * s->W);
    const Staged<int32_t> prio = h.in(pod_priority, P), grp = h.in(group, P);
    const Staged<int64_t> req = h.in(R ? res->pod_req : nullptr, P * R);
    const Staged<int64_t> node_free = h.in(R ? res->node_free : nullptr, (uint64_t)R * N);
    const NodeRulesStage rs{h, nr, rp, N};
    const Staged<ks_preemption> rows = h.out(out, P);
    const Staged<int32_t> vic = h.out(out_victims, out_victims ? P * max_victims : 0);
    const Staged<uint32_t> unres = h.out(out_unresolvable, out_unresolvable ? P : 0);
    const Staged<uint64_t> hi = h.work<uint64_t>(part_rows), lo = h.work<uint64_t>(part_rows);
    const Staged<uint32_t> cand = h.work<uint32_t>(part_rows), cnt = h.work<uint32_t>(part_rows);
    const Staged<uint32_t> unres_part = h.work<uint32_t>(part_rows);
    // the victim index's scratch: build_victim_index's block (the bound list uploaded at its start), then bound_req and
    // the R sorted request columns with their prefix sums
    const Staged<unsigned char> vx_scratch = h.work<unsigned char>(vx_bytes, 256);
    const Staged<int64_t> breq = h.work<int64_t>(N ? B * R : 0, 256);
    const Staged<int64_t> vres = h.work<int64_t>(N ? (uint64_t)R * B : 0, 256);
    const Staged<int64_t> vpre = h.work<int64_t>(N ? (uint64_t)R * B : 0, 256);
    if (const int e = h.reserve(s)) return e;
    ProfileBindArgs q{}; // k_node_rules_setup reads the NODE fields and b.N only
    q.b.N = N;
    rs.place(q, s->sms);
    CU_TRY(h.upload(st));
    VictimIndex vx{};
    FitPreemptArgs fa{R, (uint32_t)B, h.dev(req), h.dev(node_free), h.dev(grp), h.dev(rs.ncls), h.dev(rs.nrules),
                      h.dev(vres), h.dev(vpre), h.dev(unres_part)};
    if (N) {
        void* scratch = h.dev(vx_scratch);
        if (B) {
            const BoundUpload up = victim_index_inputs(scratch, B, N);
            CU_TRY(cudaMemcpyAsync(up.node, bound->node_idx, B * 4, cudaMemcpyHostToDevice, st));
            CU_TRY(cudaMemcpyAsync(up.cpu, bound->req_cpu, B * 8, cudaMemcpyHostToDevice, st));
            CU_TRY(cudaMemcpyAsync(up.mem, bound->req_mem, B * 8, cudaMemcpyHostToDevice, st));
            CU_TRY(cudaMemcpyAsync(up.prio, bound->priority, B * 4, cudaMemcpyHostToDevice, st));
            if (R) CU_TRY(cudaMemcpyAsync(h.dev(breq), bound_req, B * R * 8, cudaMemcpyHostToDevice, st));
        }
        CU_TRY(launch_node_rules(q, st));
        CU_TRY(build_victim_index(scratch, B, N, &vx, st));
        CU_TRY(build_fit_victim_index(vx, h.dev(breq), fa, N, st));
    }
    const PodView pv{h.dev(cpu), h.dev(mem), h.dev(sel), (uint32_t)P};
    const PreemptPartials part{h.dev(hi), h.dev(lo), h.dev(cand), h.dev(cnt)};
    CU_TRY(launch_fit_preempt(node_table(s), pv, h.dev(prio), vx, fa, max_victims, part, g, h.dev(rows),
                              out_victims ? h.dev(vic) : nullptr, out_unresolvable ? h.dev(unres) : nullptr, st));
    CU_TRY(h.finish(st));
    return KS_OK;
}

int ks_fit_drain_check(ks_snapshot* s, const ks_pods* pods, const int32_t* group, uint32_t n_groups,
                       const ks_node_rules* rules, const ks_bind_resources* res, const ks_drain_candidates* cand,
                       int policy, uint32_t flags, uint32_t* out_placed, int32_t* out_node_idx, int64_t* out_score,
                       uint32_t* out_refused) {
    static const ks_node_rules no_rules{};
    static const ks_bind_resources no_res{};
    DrainPlan dp;
    int rc = plan_drain(s, "ks_fit_drain_check", pods, cand, policy, flags, out_placed, out_node_idx, &dp);
    if (rc) return rc;
    const uint64_t P = dp.P, D = dp.D, G = n_groups;
    if (P && !group) return fail(KS_ERR_INVALID, "NULL group");
    if (G > KS_SPREAD_BIND_MAX_GROUPS)
        return fail(KS_ERR_RANGE, "%llu groups (at most %u)", (unsigned long long)G, KS_SPREAD_BIND_MAX_GROUPS);
    for (uint64_t p = 0; p < P; p++)
        if (group[p] < -1 || group[p] >= (int64_t)G)
            return fail(KS_ERR_INVALID, "pod %llu: group %d outside [-1, %u)", (unsigned long long)p, group[p], n_groups);
    const ks_node_rules* nr = rules ? rules : &no_rules;
    if (!res) res = &no_res;
    const uint32_t N = s->N, R = res->n_res, W = s->W;
    rc = check_bind_resources(res, P, N);
    if (rc) return rc;
    NodeRulesPlan rp;
    try {
        rc = compile_node_rules(nr, (uint32_t)G, N, &rp);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory in ks_fit_drain_check");
    }
    if (rc || D == 0) return rc;
    const uint64_t* off = cand->offset;
    const std::vector<uint32_t>&order = dp.order, &per_round = dp.per_round;
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    // pods in round order with their groups and requests, the candidates in round order, the excluded column, node_free
    // and the node rules
    const bool excl = flags & KS_DRAIN_EXCLUDE_CANDIDATES, refusals = out_refused != nullptr;
    HostStaged h;
    const auto cpu = h.in<int64_t>(nullptr, P), mem = h.in<int64_t>(nullptr, P);
    const auto sel = h.in<uint64_t>(nullptr, P * W);
    const auto grp = h.in<int32_t>(nullptr, P);
    const auto cand_node = h.in<int32_t>(nullptr, D);
    const auto pod_base = h.in<uint32_t>(nullptr, D), cand_id = h.in<uint32_t>(nullptr, D);
    const auto excluded = h.in<uint32_t>(nullptr, excl ? s->Npad / 32 : 0); // bits of the candidates' nodes
    const auto req = h.in<int64_t>(nullptr, P * R);
    const auto node_free = h.in(R ? res->node_free : nullptr, (uint64_t)R * N);
    const NodeRulesStage rs{h, nr, rp, N};
    const auto score = h.out(out_score, P);
    const auto idx = h.out(out_node_idx, P);
    const auto placed = h.out(out_placed, D);
    const auto refused = h.out(out_refused, refusals ? 4 * D : 0);
    uint64_t part_rows = 0; // node-chunk partials: the largest round needs the most
    for (uint32_t r = 0; r < dp.rounds; r++)
        part_rows = std::max<uint64_t>(part_rows, (uint64_t)fit_drain_grid(per_round[r], s->Npad, s->sms).n_chunks * per_round[r]);
    const auto ov_fc = h.work<int64_t>(P), ov_fm = h.work<int64_t>(P), part_key = h.work<int64_t>(part_rows);
    const auto ov_fr = h.work<int64_t>(P * R);
    const auto ov_node = h.work<int32_t>(P), part_idx = h.work<int32_t>(part_rows);
    const auto ov_cnt = h.work<uint32_t>(3 * D); // ov_cnt D, failed D, D zeros for the refusal pass: zeroed together
    const uint64_t DS = refusals ? D : 0;         // the stop arrays
    const auto stop_cpu = h.work<int64_t>(DS), stop_mem = h.work<int64_t>(DS), stop_req = h.work<int64_t>(DS * R);
    const auto stop_sel = h.work<uint64_t>(DS * W);
    const auto stop_grp = h.work<int32_t>(DS);
    if (const int e = h.reserve(s)) return e;
    ProfileBindArgs q{}; // k_node_rules_setup reads the NODE fields and b.N only
    q.b.N = N;
    rs.place(q, s->sms);
    int64_t *h_rc = h.host(cpu), *h_rm = h.host(mem), *h_req = h.host(req);
    uint64_t* h_sel = h.host(sel);
    int32_t *h_node = h.host(cand_node), *h_grp = h.host(grp);
    uint32_t *h_base = h.host(pod_base), *h_id = h.host(cand_id);
    for (uint64_t j = 0; j < D; j++) {
        h_node[j] = cand->node_idx[order[j]];
        h_base[j] = (uint32_t)off[order[j]];
        h_id[j] = order[j];
    }
    for (uint64_t r = 0, r0 = 0; r < dp.rounds; r0 += per_round[r], r++) // round r: pod r of the first per_round[r] candidates
        for (uint64_t j = 0; j < per_round[r]; j++) {
            const uint64_t p = off[order[j]] + r;
            h_rc[r0 + j] = pods->req_cpu[p];
            h_rm[r0 + j] = pods->req_mem[p];
            h_grp[r0 + j] = group[p];
            memcpy(h_sel + (r0 + j) * W, pods->sel + p * W, 8 * W);
            if (R) memcpy(h_req + (r0 + j) * R, res->pod_req + p * R, 8 * R);
        }
    if (excl) {
        uint32_t* h_excl = h.host(excluded);
        memset(h_excl, 0, excluded.n * 4);
        for (uint64_t d = 0; d < D; d++) h_excl[cand->node_idx[d] >> 5] |= 1u << (cand->node_idx[d] & 31);
    }
    cudaStream_t st = s->stream;
    CU_TRY(h.upload(st));
    CU_TRY(cudaMemsetAsync(h.dev(score), 0, P * 8, st));
    CU_TRY(cudaMemsetAsync(h.dev(idx), 0xff, P * 4, st));
    CU_TRY(cudaMemsetAsync(h.dev(placed), 0, D * 4, st));
    CU_TRY(cudaMemsetAsync(h.dev(ov_cnt), 0, D * 12, st));
    if (refusals) CU_TRY(cudaMemsetAsync(h.dev(refused), 0, D * 16, st));
    CU_TRY(launch_node_rules(q, st));
    DrainArgs da;
    da.cand_node = h.dev(cand_node);
    da.pod_base = h.dev(pod_base);
    da.cand_id = h.dev(cand_id);
    da.excl = excl ? h.dev(excluded) : nullptr;
    da.ov_cnt = h.dev(ov_cnt);
    da.failed = da.ov_cnt + D;
    da.ov_node = h.dev(ov_node);
    da.ov_fc = h.dev(ov_fc);
    da.ov_fm = h.dev(ov_fm);
    da.out_idx = h.dev(idx);
    da.out_score = h.dev(score);
    da.placed = h.dev(placed);
    FitDrainArgs fa{};
    fa.R = R;
    fa.P = (uint32_t)P;
    fa.node_free = h.dev(node_free);
    fa.ncls = h.dev(rs.ncls);
    fa.nrules = h.dev(rs.nrules);
    fa.ov_fr = h.dev(ov_fr);
    if (refusals) {
        fa.stop_cpu = h.dev(stop_cpu);
        fa.stop_mem = h.dev(stop_mem);
        fa.stop_sel = h.dev(stop_sel);
        fa.stop_req = h.dev(stop_req);
        fa.stop_grp = h.dev(stop_grp);
    }
    const PartialView part{h.dev(part_key), h.dev(part_idx), nullptr};
    const NodeTable nt = node_table(s);
    for (uint64_t r = 0, r0 = 0; r < dp.rounds; r0 += per_round[r], r++) {
        const PodView pv{h.dev(cpu) + r0, h.dev(mem) + r0, h.dev(sel) + r0 * W, per_round[r]};
        fa.req = h.dev(req) + r0 * R;
        fa.group = h.dev(grp) + r0;
        const DirectGrid g = fit_drain_grid(per_round[r], s->Npad, s->sms);
        const cudaError_t e = launch_fit_drain_round(nt, pv, da, fa, policy, (uint32_t)r, part, g, st);
        if (e != cudaSuccess)
            return fail(KS_ERR_CUDA, "fit drain round %llu launch failed: %s", (unsigned long long)r, cudaGetErrorString(e));
    }
    if (refusals) { // the stopped candidates' stopping pods, against their frozen overlays
        const PodView pv{fa.stop_cpu, fa.stop_mem, fa.stop_sel, (uint32_t)D};
        fa.req = fa.stop_req;
        fa.group = fa.stop_grp;
        fa.stopped = da.failed;
        fa.refused = h.dev(refused);
        DrainArgs dz = da;
        dz.failed = da.ov_cnt + 2 * D; // zeros: every slot's skip word is its destinations'
        const cudaError_t e = launch_fit_drain_refusals(nt, pv, dz, fa, fit_drain_grid((uint32_t)D, s->Npad, s->sms), st);
        if (e != cudaSuccess) return fail(KS_ERR_CUDA, "fit drain refusal pass launch failed: %s", cudaGetErrorString(e));
    }
    CU_TRY(h.finish(st));
    s->last_path = "fit_drain";
    return KS_OK;
}

int ks_fit_scaleup_estimate(ks_snapshot* s, const ks_pods* pods, const int32_t* group, uint32_t n_groups,
                            const ks_node_rules* rules, const ks_bind_resources* res, const ks_node_templates* t,
                            ks_scaleup_option* out, int32_t* out_best, int32_t* out_node, uint32_t* out_refused,
                            int64_t* out_used) {
    static const ks_node_rules no_rules{};
    static const ks_bind_resources no_res{};
    int rc = check_scaleup(s, "ks_fit_scaleup_estimate", pods, t, out, out_best);
    if (rc) return rc;
    const uint64_t P = pods->n, T = t->n, G = n_groups;
    const uint32_t W = t->label_words;
    if (P && !group) return fail(KS_ERR_INVALID, "NULL group");
    if (G > KS_SPREAD_BIND_MAX_GROUPS)
        return fail(KS_ERR_RANGE, "%llu groups (at most %u)", (unsigned long long)G, KS_SPREAD_BIND_MAX_GROUPS);
    for (uint64_t p = 0; p < P; p++)
        if (group[p] < -1 || group[p] >= (int64_t)G)
            return fail(KS_ERR_INVALID, "pod %llu: group %d outside [-1, %u)", (unsigned long long)p, group[p], n_groups);
    const ks_node_rules* nr = rules ? rules : &no_rules;
    if (!res) res = &no_res;
    const uint32_t R = res->n_res;
    rc = check_bind_resources(res, P, (uint32_t)T);
    if (rc) return rc;
    // |node_free| <= 2^52: with at most 1024 nodes per template every remainder and every out_used sum stays in int64
    for (uint64_t i = 0; i < (uint64_t)R * T; i++)
        if (res->node_free[i] < -(1ll << 52) || res->node_free[i] > (1ll << 52))
            return fail(KS_ERR_RANGE, "resource %llu, template %llu: node_free %lld outside [-2^52, 2^52]",
                        (unsigned long long)(i / T), (unsigned long long)(i % T), (long long)res->node_free[i]);
    NodeRulesPlan rp;
    try {
        rc = compile_node_rules(nr, (uint32_t)G, (uint32_t)T, &rp);
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory in ks_fit_scaleup_estimate");
    }
    if (rc) return rc;
    *out_best = -1;
    if (T == 0 || P == 0) { // nothing to pack: every row, refusal word and sum is zero
        if (T) memset(out, 0, T * sizeof(ks_scaleup_option));
        if (out_refused && P) memset(out_refused, 0, P * 16);
        if (out_used && T * R) memset(out_used, 0, T * R * 8);
        return KS_OK;
    }
    std::lock_guard<std::mutex> lk(s->mu);
    CU_TRY(cudaSetDevice(s->device));
    HostStaged h;
    const auto cpu = h.in(pods->req_cpu, P), mem = h.in(pods->req_mem, P), alloc_cpu = h.in(t->alloc_cpu, T),
               alloc_mem = h.in(t->alloc_mem, T), free_cpu = h.in(t->free_cpu, T), free_mem = h.in(t->free_mem, T);
    const auto sel = h.in(pods->sel, P * W), labels = h.in(t->labels, T * W);
    const auto max_nodes = h.in(t->max_nodes, T);
    const auto grp = h.in(group, P);
    const auto req = h.in(R ? res->pod_req : nullptr, P * R);
    const auto node_free = h.in(R ? res->node_free : nullptr, (uint64_t)R * T);
    const NodeRulesStage rs{h, nr, rp, (uint32_t)T};
    const auto rows = h.out(out, T);
    const auto refused = h.out(out_refused, out_refused ? 4 * P : 0, 16); // k_fit_scaleup_reasons stores uint4
    const auto node = h.out(out_node, out_node ? T * P : 0);
    const auto used = h.out(out_used, out_used ? T * R : 0);
    const uint32_t slots = scaleup_slots((uint32_t)T, s->sms);
    const auto scratch = h.work<uint32_t>((uint64_t)slots * 2 * P);
    if (const int e = h.reserve(s)) return e;
    ProfileBindArgs q{}; // k_node_rules_setup reads the NODE fields and b.N only
    q.b.N = (uint32_t)T;
    rs.place(q, s->sms);
    cudaStream_t st = s->stream;
    CU_TRY(h.upload(st));
    if (out_node) CU_TRY(cudaMemsetAsync(h.dev(node), 0xff, T * P * 4, st));
    CU_TRY(launch_node_rules(q, st));
    const PodView pv{h.dev(cpu), h.dev(mem), h.dev(sel), (uint32_t)P};
    ScaleupArgs a{};
    a.T = (uint32_t)T;
    a.alloc_cpu = h.dev(alloc_cpu);
    a.alloc_mem = h.dev(alloc_mem);
    a.free_cpu = h.dev(free_cpu);
    a.free_mem = h.dev(free_mem);
    a.labels = h.dev(labels);
    a.max_nodes = h.dev(max_nodes);
    a.rows = h.dev(rows);
    a.out_node = out_node ? h.dev(node) : nullptr;
    a.scratch = h.dev(scratch);
    a.slots = slots;
    FitScaleupArgs f{};
    f.R = R;
    f.req = h.dev(req);
    f.group = h.dev(grp);
    f.node_free = h.dev(node_free);
    f.ncls = h.dev(rs.ncls);
    f.nrules = h.dev(rs.nrules);
    f.used = out_used && R ? h.dev(used) : nullptr;
    f.refused = out_refused ? h.dev(refused) : nullptr;
    const cudaError_t e = launch_fit_scaleup(pv, W, a, f, st);
    if (e != cudaSuccess) return fail(KS_ERR_CUDA, "fit scale-up launch failed: %s", cudaGetErrorString(e));
    CU_TRY(h.finish(st));
    *out_best = best_template(out, T);
    s->last_path = "fit_scaleup";
    return KS_OK;
}

// ---------------------------------------------------------------------------------------------- async streaming
struct StreamItem {
    uint64_t ticket;
    int64_t rc, rm;
    uint64_t sel[KS_MAX_LABEL_WORDS];
};
struct StreamDone {
    uint64_t ticket;
    int32_t node;
    int64_t score;
};
struct ks_stream {
    ks_snapshot* snap = nullptr;
    int policy = KS_SCORE_LEFTOVER;
    uint32_t max_batch = STREAM_BATCH_MAX, W = 1;
    std::mutex mu;
    std::condition_variable cv_work, cv_idle;
    std::deque<StreamItem> in;
    std::deque<StreamDone> out;
    uint64_t submitted = 0, finished = 0, batches = 0, rounds = 0, max_seen = 0;
    bool stop = false;
    bool dead = false; // the dispatcher thread could not start working (out of memory)
    int error = KS_OK;
    std::thread worker;
};

static void stream_worker(ks_stream* q) {
    std::vector<int64_t> rc, rm, score;
    std::vector<uint64_t> sel, tickets;
    std::vector<int32_t> idx;
    try { // every per-batch resize below stays within these capacities: the loop itself never allocates
        rc.reserve(q->max_batch);
        rm.reserve(q->max_batch);
        score.reserve(q->max_batch);
        idx.reserve(q->max_batch);
        tickets.reserve(q->max_batch);
        sel.reserve((size_t)q->max_batch * q->W);
    } catch (...) { // no dispatcher: submissions are answered with the error code by ks_stream_poll / ks_stream_flush
        std::lock_guard<std::mutex> lk(q->mu);
        q->error = KS_ERR_NOMEM;
        q->dead = true;
        q->cv_idle.notify_all();
        return;
    }
    for (;;) {
        {
            std::unique_lock<std::mutex> lk(q->mu);
            q->cv_work.wait(lk, [&] { return q->stop || !q->in.empty(); });
            if (q->stop) return;
            const size_t m = std::min<size_t>(q->in.size(), q->max_batch);
            rc.resize(m);
            rm.resize(m);
            sel.resize(m * q->W);
            tickets.resize(m);
            for (size_t k = 0; k < m; k++) { // everything that has arrived, in arrival order
                const StreamItem& it = q->in.front();
                rc[k] = it.rc;
                rm[k] = it.rm;
                tickets[k] = it.ticket;
                for (uint32_t w = 0; w < q->W; w++) sel[k * q->W + w] = it.sel[w];
                q->in.pop_front();
            }
        }
        const size_t m = rc.size();
        idx.assign(m, -1);
        score.assign(m, 0);
        uint32_t rounds = 0;
        ks_pods kp{m, rc.data(), rm.data(), sel.data(), KS_MEM_HOST};
        const int e = ks_stream_bind(q->snap, &kp, q->policy, idx.data(), score.data(), &rounds);
        {
            std::lock_guard<std::mutex> lk(q->mu);
            if (e) q->error = e;
            try {
                for (size_t k = 0; k < m; k++) q->out.push_back(StreamDone{tickets[k], e ? -1 : idx[k], e ? 0 : score[k]});
            } catch (...) { // results that could not be queued are lost; the poller gets the error code
                q->error = KS_ERR_NOMEM;
            }
            q->finished += m;
            q->batches++;
            q->rounds += rounds;
            q->max_seen = std::max<uint64_t>(q->max_seen, m);
        }
        q->cv_idle.notify_all();
    }
}

int ks_stream_open(ks_snapshot* s, int policy, uint32_t max_batch, ks_stream** out) {
    if (!s || !out) return fail(KS_ERR_INVALID, "NULL argument");
    if (!policy_valid(policy)) return fail(KS_ERR_INVALID, "bad policy");
    ks_stream* q = new (std::nothrow) ks_stream();
    if (!q) return fail(KS_ERR_NOMEM, "out of host memory");
    q->snap = s;
    q->policy = policy;
    q->W = s->W;
    q->max_batch = max_batch == 0 ? STREAM_BATCH_MAX : std::min<uint32_t>(max_batch, STREAM_BATCH_MAX);
    try {
        q->worker = std::thread(stream_worker, q);
    } catch (...) {
        delete q;
        return fail(KS_ERR_NOMEM, "cannot start the dispatcher thread");
    }
    *out = q;
    return KS_OK;
}

int ks_stream_submit(ks_stream* q, uint64_t n, const int64_t* req_cpu, const int64_t* req_mem, const uint64_t* sel,
                     const uint64_t* tickets) {
    if (!q || (n && (!req_cpu || !req_mem || !sel || !tickets))) return fail(KS_ERR_INVALID, "NULL argument");
    if (n == 0) return KS_OK;
    // checked here, so that one bad pod fails its own submit and not the dispatcher batch it would have joined
    const int rc = check_commit_requests(n, req_cpu, req_mem);
    if (rc) return rc;
    try {
        std::lock_guard<std::mutex> lk(q->mu);
        for (uint64_t i = 0; i < n; i++) {
            StreamItem it;
            it.ticket = tickets[i];
            it.rc = req_cpu[i];
            it.rm = req_mem[i];
            for (uint32_t w = 0; w < q->W; w++) it.sel[w] = sel[i * q->W + w];
            q->in.push_back(it);
        }
        q->submitted += n;
    } catch (...) {
        return fail(KS_ERR_NOMEM, "out of host memory");
    }
    q->cv_work.notify_one();
    return KS_OK;
}

int ks_stream_poll(ks_stream* q, uint64_t max, uint64_t* out_ticket, int32_t* out_node_idx, int64_t* out_score, uint64_t* out_n) {
    if (!q || !out_n || (max && (!out_ticket || !out_node_idx))) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(q->mu);
    uint64_t k = 0;
    while (k < max && !q->out.empty()) {
        const StreamDone& d = q->out.front();
        out_ticket[k] = d.ticket;
        out_node_idx[k] = d.node;
        if (out_score) out_score[k] = d.score;
        q->out.pop_front();
        k++;
    }
    *out_n = k;
    if (q->error) {
        const int e = q->error;
        q->error = KS_OK;
        return e; // ks_last_error() of the dispatcher thread is not visible here: the code says what failed
    }
    return KS_OK;
}

int ks_stream_flush(ks_stream* q) {
    if (!q) return fail(KS_ERR_INVALID, "NULL argument");
    std::unique_lock<std::mutex> lk(q->mu);
    q->cv_idle.wait(lk, [&] { return q->dead || q->finished == q->submitted; });
    if (q->dead) return fail(KS_ERR_NOMEM, "the stream's dispatcher thread is not running (out of host memory)");
    return KS_OK;
}

int ks_stream_stats(ks_stream* q, uint64_t* batches, uint64_t* rounds, uint64_t* max_batch_seen) {
    if (!q) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(q->mu);
    if (batches) *batches = q->batches;
    if (rounds) *rounds = q->rounds;
    if (max_batch_seen) *max_batch_seen = q->max_seen;
    return KS_OK;
}

void ks_stream_close(ks_stream* q) {
    if (!q) return;
    {
        std::lock_guard<std::mutex> lk(q->mu);
        q->stop = true;
    }
    q->cv_work.notify_all();
    if (q->worker.joinable()) q->worker.join();
    delete q;
}

} // extern "C"
