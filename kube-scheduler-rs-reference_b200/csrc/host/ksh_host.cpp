// ksh_host.cpp — host layer over Pod/Node objects (include/ksched_host.h): quantity parsing, packing into
// SoA int64 + label bit columns, and the mirror of check_node_validity / select_node_for_pod / reconcile.
// It only packs and dispatches: every predicate is evaluated by the CUDA core (ks_* in ksched.h).
// Built for cluster scale: strings are interned once (no per-lookup allocation), label pairs and node names are
// integers afterwards, node/pod events cost O(labels of the object), and the bulk calls (LIST results, pod
// batches) are parsed by all host threads with results identical to the single-thread order.
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <algorithm>
#include <array>
#include <atomic>
#include <cstdlib>
#include <functional>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../../include/ksched_host.h"

extern "C" void ks__set_error(const char* msg); // defined in ks_api.cu (not part of the public ABI)
// ks_explain, ks_select_topk, ks_preempt, ks_gang_bind, ks_drain_check and ks_scaleup_estimate are defined by the CUDA
// core in the same library.  The references are weak so that this file still links with device stand-ins that only
// provide the older ks_* entries (tests/native); ksh_explain_pods, ksh_rank_nodes, ksh_preempt_pods, ksh_reconcile_gangs,
// ksh_drain_nodes, ksh_scaleup_estimate, ksh_place_replicas and ksh_place_replicas_spread (and _multi) then report
// KS_ERR_NO_DEVICE.
#pragma weak ks_explain
#pragma weak ks_select_topk
#pragma weak ks_preempt
#pragma weak ks_gang_bind
#pragma weak ks_drain_check
#pragma weak ks_scaleup_estimate
#pragma weak ks_fit_scaleup_estimate
#pragma weak ks_place_replicas
#pragma weak ks_place_replicas_spread
#pragma weak ks_place_replicas_spread_multi
#pragma weak ks_spread_bind
#pragma weak ks_affinity_bind
#pragma weak ks_profile_bind
#pragma weak ks_node_bind
#pragma weak ks_fit_bind
#pragma weak ks_gang_fit_bind
#pragma weak ks_fit_preempt
#pragma weak ks_fit_drain_check

namespace {

int fail(int code, const std::string& msg) {
    ks__set_error(msg.c_str());
    return code;
}

// Nothing may throw across the C ABI (ksched_host.h): every extern "C" entry point is a function-try-block ending here
#define KSH_CATCH                                                                                   \
    catch (const std::bad_alloc&) { return fail(KS_ERR_NOMEM, "out of host memory in the host layer"); } \
    catch (...) { return fail(KS_ERR_INVALID, "unexpected C++ exception in the host layer"); }

typedef unsigned __int128 u128;

// Kubernetes quantity: sign? digits [. digits] (binarySI | decimalSI | decimalExponent)?
// Result = value * 10^unit_shift as an exact integer (unit_shift 3 -> milli-units, 0 -> units).
int parse_quantity(const char* s, int unit_shift, int64_t* out) {
    if (!s) return KS_ERR_PARSE;
    size_t i = 0;
    bool neg = false;
    if (s[i] == '+' || s[i] == '-') neg = s[i++] == '-';
    u128 mant = 0;
    int int_digits = 0, frac_digits = 0;
    const u128 cap = (u128)1 << 96;
    { // the first 18 digits fit 64-bit arithmetic: every realistic quantity takes only this loop
        uint64_t m64 = 0;
        while (int_digits < 18 && s[i] >= '0' && s[i] <= '9') {
            m64 = m64 * 10 + (unsigned)(s[i++] - '0');
            int_digits++;
        }
        mant = m64;
    }
    while (s[i] >= '0' && s[i] <= '9') {
        if (mant >= cap) return KS_ERR_RANGE;
        mant = mant * 10 + (unsigned)(s[i++] - '0');
        int_digits++;
    }
    if (s[i] == '.') {
        i++;
        while (s[i] >= '0' && s[i] <= '9') {
            if (mant >= cap) return KS_ERR_RANGE;
            mant = mant * 10 + (unsigned)(s[i++] - '0');
            frac_digits++;
        }
    }
    if (int_digits + frac_digits == 0) return KS_ERR_PARSE;
    int p10 = -frac_digits, p2 = 0;
    const char c = s[i];
    if (c == '\0') {
    } else if (s[i + 1] == 'i' && s[i + 2] == '\0' && std::strchr("KMGTPE", c)) {
        p2 = 10 * (int)(std::strchr("KMGTPE", c) - "KMGTPE" + 1);
        i += 2;
    } else if ((c == 'e' || c == 'E') && s[i + 1] != '\0' &&
               ((s[i + 1] >= '0' && s[i + 1] <= '9') ||
                ((s[i + 1] == '+' || s[i + 1] == '-') && s[i + 2] >= '0' && s[i + 2] <= '9'))) {
        i++;
        bool eneg = false;
        if (s[i] == '+' || s[i] == '-') eneg = s[i++] == '-';
        int e = 0;
        while (s[i] >= '0' && s[i] <= '9') {
            e = e * 10 + (s[i++] - '0');
            if (e > 4000) return KS_ERR_RANGE;
        }
        p10 += eneg ? -e : e;
    } else {
        static const char suf[] = "numkMGTPE";
        static const int exp[] = {-9, -6, -3, 3, 6, 9, 12, 15, 18};
        const char* f = c ? std::strchr(suf, c) : nullptr;
        if (!f) return KS_ERR_PARSE;
        p10 += exp[f - suf];
        i++;
    }
    if (s[i] != '\0') return KS_ERR_PARSE;
    p10 += unit_shift;
    u128 v = mant;
    if (v != 0) {
        if (p2) {
            if (v >= (cap >> p2)) return KS_ERR_RANGE;
            v <<= p2;
        }
        while (p10 > 0) {
            if (v >= cap) return KS_ERR_RANGE;
            v *= 10;
            p10--;
        }
        while (p10 < 0) {
            if (v % 10 != 0) return KS_ERR_INEXACT;
            v /= 10;
            p10++;
        }
    }
    if (v > (u128)INT64_MAX) return KS_ERR_RANGE;
    *out = neg ? -(int64_t)v : (int64_t)v;
    return KS_OK;
}

const char* kv_find(const ks_kv* kv, uint32_t n, const char* key) {
    for (uint32_t i = 0; i < n; i++)
        if (kv[i].key && std::strcmp(kv[i].key, key) == 0) return kv[i].val;
    return nullptr;
}

void json_escape(std::string& out, const char* s) {
    for (; s && *s; s++) {
        const unsigned char c = (unsigned char)*s;
        if (c == '"' || c == '\\') {
            out.push_back('\\');
            out.push_back((char)c);
        } else if (c < 0x20) {
            char buf[8];
            std::snprintf(buf, sizeof(buf), "\\u%04x", c);
            out += buf;
        } else {
            out.push_back((char)c);
        }
    }
}

} // namespace

// ---- string interning: (a, sep, b) byte strings -> dense ids in insertion order; lookups allocate nothing ----
static inline uint64_t hash_bytes(uint64_t h, const char* s, size_t n) {
    for (size_t i = 0; i < n; i++) h = (h ^ (unsigned char)s[i]) * 0x100000001B3ull; // FNV-1a
    return h;
}
static inline uint64_t hash2(const char* a, size_t la, char sep, const char* b, size_t lb) {
    uint64_t h = hash_bytes(0xCBF29CE484222325ull, a, la);
    h = (h ^ (unsigned char)sep) * 0x100000001B3ull;
    h = hash_bytes(h, b, lb);
    h ^= h >> 32; // the table index uses the low bits
    return h;
}

struct Interner {
    struct Ent {
        uint64_t h;
        uint64_t off;
        uint32_t len;
    };
    std::vector<char> arena; // every string stored NUL-terminated
    std::vector<Ent> ents;
    std::vector<uint32_t> slots; // open addressing, linear probing; EMPTY = free
    static constexpr uint32_t EMPTY = 0xFFFFFFFFu;

    void clear() {
        arena.clear();
        ents.clear();
        slots.clear();
    }
    size_t size() const { return ents.size(); }
    const char* str(uint32_t id) const { return arena.data() + ents[id].off; }
    bool equal(const Ent& e, uint64_t h, const char* a, size_t la, char sep, const char* b, size_t lb) const {
        if (e.h != h || e.len != la + 1 + lb) return false;
        const char* s = arena.data() + e.off;
        return std::memcmp(s, a, la) == 0 && s[la] == sep && std::memcmp(s + la + 1, b, lb) == 0;
    }
    int64_t find_h(uint64_t h, const char* a, size_t la, char sep, const char* b, size_t lb) const {
        if (slots.empty()) return -1;
        const size_t mask = slots.size() - 1;
        for (size_t i = h & mask;; i = (i + 1) & mask) {
            const uint32_t id = slots[i];
            if (id == EMPTY) return -1;
            if (equal(ents[id], h, a, la, sep, b, lb)) return id;
        }
    }
    int64_t find(const char* a, char sep, const char* b) const {
        const size_t la = std::strlen(a), lb = std::strlen(b);
        return find_h(hash2(a, la, sep, b, lb), a, la, sep, b, lb);
    }
    void grow() {
        const size_t cap = slots.empty() ? 64 : slots.size() * 2;
        slots.assign(cap, EMPTY);
        for (uint32_t id = 0; id < ents.size(); id++) {
            size_t i = ents[id].h & (cap - 1);
            while (slots[i] != EMPTY) i = (i + 1) & (cap - 1);
            slots[i] = id;
        }
    }
    uint32_t intern_h(uint64_t h, const char* a, size_t la, char sep, const char* b, size_t lb) {
        const int64_t f = find_h(h, a, la, sep, b, lb);
        if (f >= 0) return (uint32_t)f;
        if ((ents.size() + 1) * 2 > slots.size()) grow();
        const uint32_t id = (uint32_t)ents.size();
        ents.push_back({h, (uint64_t)arena.size(), (uint32_t)(la + 1 + lb)});
        arena.insert(arena.end(), a, a + la);
        arena.push_back(sep);
        arena.insert(arena.end(), b, b + lb);
        arena.push_back('\0');
        const size_t mask = slots.size() - 1;
        size_t i = h & mask;
        while (slots[i] != EMPTY) i = (i + 1) & mask;
        slots[i] = id;
        return id;
    }
    uint32_t intern(const char* a, char sep, const char* b) {
        const size_t la = std::strlen(a), lb = std::strlen(b);
        return intern_h(hash2(a, la, sep, b, lb), a, la, sep, b, lb);
    }
};

static inline const char* nz(const char* s) { return s ? s : ""; }

// ---- bound pods keyed by "namespace/name": key hash -> position, with erase (positions move on swap-remove) ----
struct PosTable {
    // slot = (high 32 bits of the key hash) << 32 | (position + 2); low word 0 = empty, 1 = tombstone
    std::vector<uint64_t> slots;
    size_t used = 0; // live + tombstones
    void clear() {
        slots.clear();
        used = 0;
    }
};

// One quantity of a scalar resource (numbered by ksh_context::res_id).  A quantity that does not parse, or a pod's sum
// over its containers that leaves int64, is kept with its error rather than rejected, so that every call that ignores
// these resources behaves as before; a call that needs the resource reports it (ext_error).
enum : uint8_t { EXT_OK = 0, EXT_PARSE = 1, EXT_OVERFLOW = 2 };
struct ExtQty {
    uint32_t res;
    uint8_t err; // EXT_OK, EXT_PARSE or EXT_OVERFLOW; v is meaningful only with EXT_OK
    int64_t v;
};

struct ksh_context {
    ks_snapshot* snap = nullptr;
    uint32_t N = 0;
    // nodes: names are interned once; name id -> current index (-1 = gone), index -> name id
    Interner names;
    std::vector<int32_t> nameid2idx;
    std::vector<uint32_t> idx2nameid;
    std::vector<int64_t> alloc_cpu, alloc_mem;
    // label pairs "key\0value" interned to pair ids; per pair: how many nodes carry it, and its dictionary bit
    Interner pairs;
    std::vector<uint32_t> pair_refcnt;
    std::vector<int32_t> pair_bit;            // -1 = no selector has named this pair yet
    std::vector<uint32_t> bit2pair;           // dictionary, in order of assignment
    std::vector<std::vector<uint32_t>> node_pids; // per node: pair ids of its labels
    uint32_t W = 1;
    // bound pods (the LIST results of predicates.rs:21-34), swap-remove on delete
    std::vector<int32_t> bnode;
    std::vector<int64_t> bcpu, bmem;
    std::vector<uint64_t> bhash;  // hash of "ns/name"; 0 with blen 0 = anonymous pod, not tracked
    std::vector<uint64_t> boff;   // key bytes in bkeys
    std::vector<uint32_t> blen;
    std::vector<int32_t> bprio;   // spec.priority (ksh_context_set_pod_priorities), 0 until set
    std::vector<char> bkeys;
    PosTable btab;
    uint64_t live_pairs = 0;     // pairs carried by at least one node
    uint64_t live_key_bytes = 0; // bytes of bkeys that belong to current rows
    // scratch of the bulk calls, kept between calls (fresh pages are expensive to fault in)
    std::vector<int32_t> tmp_node;
    std::vector<int64_t> tmp_cpu, tmp_mem;
    std::vector<uint64_t> tmp_hash;
    std::vector<uint32_t> tmp_len;
    std::vector<int64_t> pk_cpu, pk_mem; // packed form of the last batch a device call packed (pack_batch)
    std::vector<uint64_t> pk_sel;
    bool dirty = true; // device snapshot must be re-uploaded
    // spec.taints by node name (ksh_context_set_node_taints): key, value, effect
    std::unordered_map<std::string, std::vector<std::array<std::string, 3>>> taints;
    // scalar resources other than cpu and memory (ksh_reconcile_fit, DESIGN.md 5r): names numbered once; per node its
    // allocatable quantities, per bound row its non-zero requests (empty for a pod without extended requests)
    std::unordered_map<std::string, uint32_t> res_id;
    std::vector<std::string> res_name;
    std::vector<std::vector<ExtQty>> node_ext; // [N]
    std::vector<std::vector<ExtQty>> bext;     // per bound row, in step with bnode
    // one lock per context: every ksh_* entry that takes a context holds it for the whole call (entries call each other)
    mutable std::recursive_mutex mu;
};

static uint32_t words_for_bits(uint32_t real_bits) {
    // +1: the last bit of the last word is the shared "no node carries this pair" bit
    uint32_t w = 1;
    while ((uint64_t)w * 64 < (uint64_t)real_bits + 1) w <<= 1;
    return w;
}

// ---- threads ----
static unsigned host_threads() {
    static const unsigned t = [] {
        if (const char* e = std::getenv("KSH_THREADS")) {
            const int v = std::atoi(e);
            if (v > 0) return (unsigned)std::min(v, 256);
        }
        const unsigned hc = std::thread::hardware_concurrency();
        return std::max(1u, std::min(hc ? hc : 1u, 32u));
    }();
    return t;
}

// f(thread, begin, end) over [0,n) in contiguous ascending ranges: concatenating per-thread results in thread order
// reproduces the serial order
template <class F>
static unsigned parallel_ranges(uint64_t n, uint64_t min_per_thread, F f) {
    unsigned T = (unsigned)std::min<uint64_t>(host_threads(), std::max<uint64_t>(1, n / std::max<uint64_t>(1, min_per_thread)));
    if (T <= 1) {
        f(0u, (uint64_t)0, n);
        return 1;
    }
    std::vector<std::thread> th;
    th.reserve(T - 1);
    const uint64_t per = (n + T - 1) / T;
    std::atomic<bool> oom{false}; // an exception must not leave a worker thread: it is re-raised after the join
    for (unsigned t = 1; t < T; t++)
        th.emplace_back([=, &f, &oom] {
            try {
                f(t, std::min(n, t * per), std::min(n, (t + 1) * per));
            } catch (...) {
                oom = true;
            }
        });
    try {
        f(0u, (uint64_t)0, std::min(n, per));
    } catch (...) {
        oom = true;
    }
    for (auto& x : th) x.join();
    if (oom) throw std::bad_alloc();
    return T;
}

struct alignas(128) RangeError { // first failure of a range (ranges stop at their first failure); one cache line pair each
    int rc = KS_OK;
    std::string msg;
};
static int first_error(const std::vector<RangeError>& errs) {
    for (const RangeError& e : errs)
        if (e.rc) return fail(e.rc, e.msg);
    return KS_OK;
}

// ---- parsing without touching the caller-visible error string (usable from worker threads) ----
static int parse_cpu(const char* q, int64_t* out, std::string* err) {
    const int rc = parse_quantity(q, 3, out);
    if (rc) *err = std::string("cannot convert cpu quantity '") + (q ? q : "(null)") + "' to integer millicores";
    return rc;
}
static int parse_mem(const char* q, int64_t* out, std::string* err) {
    const int rc = parse_quantity(q, 0, out);
    if (rc) *err = std::string("cannot convert memory quantity '") + (q ? q : "(null)") + "' to integer bytes";
    return rc;
}

// src/util.rs:54-75: sum of resources.requests over spec.containers only (no initContainers, no limits)
static int total_pod_resources(const ks_pod_obj* pod, int64_t* cpu, int64_t* mem, std::string* err) {
    int64_t c = 0, m = 0;
    if (pod->has_spec) {
        for (uint32_t i = 0; i < pod->n_containers; i++) {
            const ks_container_obj& ct = pod->containers[i];
            if (!ct.has_requests) continue;
            if (const char* q = kv_find(ct.requests, ct.n_requests, "cpu")) {
                int64_t v;
                const int rc = parse_cpu(q, &v, err); // reference: .expect("invalid pod spec: cpu request")
                if (rc) return rc;
                if (__builtin_add_overflow(c, v, &c)) return *err = "cpu request sum overflows", KS_ERR_RANGE;
            }
            if (const char* q = kv_find(ct.requests, ct.n_requests, "memory")) {
                int64_t v;
                const int rc = parse_mem(q, &v, err);
                if (rc) return rc;
                if (__builtin_add_overflow(m, v, &m)) return *err = "memory request sum overflows", KS_ERR_RANGE;
            }
        }
    }
    if (c > KS_MAX_CPU_MILLI || c < -KS_MAX_CPU_MILLI || m > KS_MAX_MEM_BYTES || m < -KS_MAX_MEM_BYTES)
        return *err = "pod requests outside +-2^36 millicores / +-2^55 bytes", KS_ERR_RANGE;
    *cpu = c;
    *mem = m;
    return KS_OK;
}

// allocatable of one node; mirrors src/predicates.rs:27-32
static int parse_node_allocatable(const ks_node_obj& nd, int64_t* ac, int64_t* am, std::string* err) {
    *ac = 0;
    *am = 0; // status/allocatable None => PodResources::new() = (0,0)   (predicates.rs:27-28)
    if (!nd.has_allocatable) return KS_OK;
    const std::string name = nz(nd.name);
    const char* q = kv_find(nd.allocatable, nd.n_allocatable, "cpu");
    if (!q) return *err = "node '" + name + "': allocatable has no cpu (reference panics, predicates.rs:29)", KS_ERR_MISSING;
    int rc = parse_cpu(q, ac, err);
    if (rc) return rc;
    q = kv_find(nd.allocatable, nd.n_allocatable, "memory");
    if (!q) return *err = "node '" + name + "': allocatable has no memory (reference panics, predicates.rs:30)", KS_ERR_MISSING;
    rc = parse_mem(q, am, err);
    if (rc) return rc;
    if (*ac > KS_MAX_CPU_MILLI || *ac < -KS_MAX_CPU_MILLI || *am > KS_MAX_MEM_BYTES || *am < -KS_MAX_MEM_BYTES)
        return *err = "node '" + name + "': allocatable out of range", KS_ERR_RANGE;
    return KS_OK;
}

// ---- label pairs ----
static uint32_t intern_pair(ksh_context* c, uint64_t h, const char* k, size_t lk, const char* v, size_t lv) {
    const uint32_t pid = c->pairs.intern_h(h, k, lk, '\0', v, lv);
    if (pid == c->pair_refcnt.size()) {
        c->pair_refcnt.push_back(0);
        c->pair_bit.push_back(-1);
    }
    return pid;
}

static void node_pairs_release(ksh_context* c, uint32_t idx) {
    for (uint32_t pid : c->node_pids[idx])
        if (--c->pair_refcnt[pid] == 0) c->live_pairs--;
    c->node_pids[idx].clear();
}

static void node_pairs_set(ksh_context* c, uint32_t idx, const ks_node_obj& nd) {
    std::vector<uint32_t>& v = c->node_pids[idx];
    if (!nd.has_labels) return;
    for (uint32_t l = 0; l < nd.n_labels; l++) {
        const char *k = nz(nd.labels[l].key), *val = nz(nd.labels[l].val);
        const size_t lk = std::strlen(k), lv = std::strlen(val);
        const uint32_t pid = intern_pair(c, hash2(k, lk, '\0', val, lv), k, lk, val, lv);
        if (std::find(v.begin(), v.end(), pid) != v.end()) continue; // a map has each key once; be safe
        v.push_back(pid);
        if (c->pair_refcnt[pid]++ == 0) c->live_pairs++;
    }
}

// A long-running host sees label values, node names and pods come and go; what the interners and the key arena
// keep for objects that no longer exist is reclaimed once it outweighs the live part.
static constexpr size_t GC_SLACK = 1024;

static void gc_pairs(ksh_context* c) {
    if (c->pairs.size() <= 2 * c->live_pairs + GC_SLACK) return;
    Interner fresh;
    std::vector<uint32_t> refcnt;
    std::vector<int32_t> bit;
    std::vector<uint32_t> remap(c->pairs.size(), 0xFFFFFFFFu);
    auto move_pair = [&](uint32_t pid) {
        if (remap[pid] != 0xFFFFFFFFu) return remap[pid];
        const Interner::Ent& e = c->pairs.ents[pid];
        const char* k = c->pairs.str(pid);
        const size_t lk = std::strlen(k);
        const uint32_t id = fresh.intern_h(e.h, k, lk, '\0', k + lk + 1, e.len - lk - 1);
        refcnt.push_back(c->pair_refcnt[pid]);
        bit.push_back(c->pair_bit[pid]);
        return remap[pid] = id;
    };
    for (uint32_t& pid : c->bit2pair) pid = move_pair(pid); // dictionary entries survive, stale ones included
    for (auto& v : c->node_pids)
        for (uint32_t& pid : v) pid = move_pair(pid);
    c->pairs = std::move(fresh);
    c->pair_refcnt.swap(refcnt);
    c->pair_bit.swap(bit);
}

static void gc_names(ksh_context* c) {
    if (c->names.size() <= 2 * (size_t)c->N + GC_SLACK) return;
    Interner fresh;
    std::vector<int32_t> id2idx;
    for (uint32_t i = 0; i < c->N; i++) {
        const uint32_t old = c->idx2nameid[i];
        const char* name = c->names.str(old);
        const uint32_t id = fresh.intern_h(c->names.ents[old].h, name, std::strlen(name), '\0', "", 0);
        if (id == id2idx.size()) id2idx.push_back((int32_t)i); // rows are visited in index order: the first row of a name wins
        c->idx2nameid[i] = id;
    }
    c->names = std::move(fresh);
    c->nameid2idx.swap(id2idx);
}

static void gc_bound_keys(ksh_context* c) {
    if (c->bkeys.size() <= 2 * c->live_key_bytes + 64 * GC_SLACK) return;
    std::vector<char> fresh;
    fresh.reserve(c->live_key_bytes);
    for (size_t pos = 0; pos < c->bnode.size(); pos++) {
        if (c->blen[pos] == 0) continue;
        const uint64_t off = fresh.size();
        fresh.insert(fresh.end(), c->bkeys.begin() + (ptrdiff_t)c->boff[pos], c->bkeys.begin() + (ptrdiff_t)(c->boff[pos] + c->blen[pos]));
        c->boff[pos] = off;
    }
    c->bkeys.swap(fresh);
}

// Dictionary bits of pairs that no node carries any more are dead weight (a selector naming such a pair is
// infeasible everywhere either way); they are dropped, and the rest renumbered in order, when space is needed.
static void compact_dictionary(ksh_context* c) {
    std::vector<uint32_t> kept;
    for (uint32_t pid : c->bit2pair) {
        if (c->pair_refcnt[pid] > 0) {
            c->pair_bit[pid] = (int32_t)kept.size();
            kept.push_back(pid);
        } else {
            c->pair_bit[pid] = -1;
        }
    }
    if (kept.size() != c->bit2pair.size()) c->dirty = true;
    c->bit2pair.swap(kept);
}

static int assign_bit(ksh_context* c, uint32_t pid) {
    if (c->pair_bit[pid] >= 0) return KS_OK;
    if (words_for_bits((uint32_t)c->bit2pair.size() + 1) > KS_MAX_LABEL_WORDS) {
        compact_dictionary(c);
        if (words_for_bits((uint32_t)c->bit2pair.size() + 1) > KS_MAX_LABEL_WORDS)
            return fail(KS_ERR_RANGE, "more than 511 distinct (key,value) pairs referenced by selectors");
    }
    c->pair_bit[pid] = (int32_t)c->bit2pair.size();
    c->bit2pair.push_back(pid);
    c->dirty = true;
    return KS_OK;
}

static void update_words(ksh_context* c) {
    const uint32_t w = words_for_bits((uint32_t)c->bit2pair.size());
    if (w != c->W) {
        c->W = w;
        c->dirty = true;
    }
}

// node label words [N*W] under the current dictionary
static void fill_label_words(const ksh_context* c, uint64_t* lab) {
    std::memset(lab, 0, (size_t)c->N * c->W * sizeof(uint64_t));
    for (uint32_t n = 0; n < c->N; n++)
        for (uint32_t pid : c->node_pids[n]) {
            const int32_t bit = c->pair_bit[pid];
            if (bit >= 0) lab[(size_t)n * c->W + ((uint32_t)bit >> 6)] |= 1ull << (bit & 63);
        }
}

// ---- bound pods ----
static inline uint64_t pod_key_hash(const ks_pod_obj* pod, size_t* lns, size_t* lname) {
    const char *ns = nz(pod->ns), *name = nz(pod->name);
    *lns = std::strlen(ns);
    *lname = std::strlen(name);
    return hash2(ns, *lns, '/', name, *lname);
}

static bool bkey_equal(const ksh_context* c, size_t pos, uint64_t h, const ks_pod_obj* pod, size_t lns, size_t lname) {
    if (c->bhash[pos] != h || c->blen[pos] != lns + 1 + lname) return false;
    const char* s = c->bkeys.data() + c->boff[pos];
    return std::memcmp(s, nz(pod->ns), lns) == 0 && s[lns] == '/' && std::memcmp(s + lns + 1, nz(pod->name), lname) == 0;
}

static inline uint64_t btab_word(uint64_t h, size_t pos) { return (h & 0xFFFFFFFF00000000ull) | (uint32_t)(pos + 2); }
static inline uint32_t slot_low(uint64_t s) { return (uint32_t)s; }

static void btab_rebuild(ksh_context* c, size_t want_live) {
    size_t cap = 64;
    while (cap < want_live * 2 + 2) cap *= 2;
    c->btab.slots.assign(cap, 0);
    c->btab.used = 0;
    for (size_t pos = 0; pos < c->bnode.size(); pos++) {
        if (c->blen[pos] == 0) continue;
        size_t i = c->bhash[pos] & (cap - 1);
        while (c->btab.slots[i] != 0) i = (i + 1) & (cap - 1);
        c->btab.slots[i] = btab_word(c->bhash[pos], pos);
        c->btab.used++;
    }
}

static int64_t btab_find_slot(const ksh_context* c, uint64_t h, const ks_pod_obj* pod, size_t lns, size_t lname) {
    if (c->btab.slots.empty()) return -1;
    const size_t mask = c->btab.slots.size() - 1;
    for (size_t i = h & mask;; i = (i + 1) & mask) {
        const uint64_t s = c->btab.slots[i];
        if (s == 0) return -1;
        if (slot_low(s) >= 2 && (s >> 32) == (h >> 32) && bkey_equal(c, slot_low(s) - 2, h, pod, lns, lname)) return (int64_t)i;
    }
}

static int64_t btab_slot_of_pos(const ksh_context* c, size_t pos) {
    if (c->btab.slots.empty()) return -1;
    const size_t mask = c->btab.slots.size() - 1;
    for (size_t i = c->bhash[pos] & mask;; i = (i + 1) & mask) {
        const uint64_t s = c->btab.slots[i];
        if (s == 0) return -1;
        if (slot_low(s) == pos + 2) return (int64_t)i;
    }
}

static void bound_erase(ksh_context* c, size_t pos);

static uint32_t res_id(ksh_context* c, const char* name) {
    const auto it = c->res_id.find(name);
    if (it != c->res_id.end()) return it->second;
    const uint32_t id = (uint32_t)c->res_name.size();
    c->res_name.emplace_back(name);
    c->res_id.emplace(name, id);
    return id;
}

static inline bool cpu_or_memory(const char* k) { return !std::strcmp(k, "cpu") || !std::strcmp(k, "memory"); }

// The pod's requests of every resource but cpu and memory, summed over spec.containers as total_pod_resources sums cpu
// and memory; zero sums dropped
static std::vector<ExtQty> pod_ext(ksh_context* c, const ks_pod_obj* pod) {
    std::vector<ExtQty> out;
    if (!pod->has_spec) return out;
    for (uint32_t i = 0; i < pod->n_containers; i++) {
        const ks_container_obj& ct = pod->containers[i];
        if (!ct.has_requests) continue;
        for (uint32_t j = 0; j < ct.n_requests; j++) {
            const ks_kv& kv = ct.requests[j];
            if (!kv.key || cpu_or_memory(kv.key)) continue;
            int64_t v = 0;
            const uint8_t err = parse_quantity(kv.val, 0, &v) != KS_OK ? EXT_PARSE : EXT_OK;
            const uint32_t r = res_id(c, kv.key);
            auto it = std::find_if(out.begin(), out.end(), [r](const ExtQty& e) { return e.res == r; });
            if (it == out.end()) out.push_back({r, err, err ? 0 : v});
            else if (err) it->err = it->err ? it->err : err;
            else if (!it->err && __builtin_add_overflow(it->v, v, &it->v)) it->err = EXT_OVERFLOW;
        }
    }
    out.erase(std::remove_if(out.begin(), out.end(), [](const ExtQty& e) { return !e.err && e.v == 0; }), out.end());
    return out;
}

// The node's allocatable quantities of every resource but cpu and memory ("pods" included), the first of a repeated key
static std::vector<ExtQty> node_ext(ksh_context* c, const ks_node_obj& nd) {
    std::vector<ExtQty> out;
    if (!nd.has_allocatable) return out;
    for (uint32_t j = 0; j < nd.n_allocatable; j++) {
        const ks_kv& kv = nd.allocatable[j];
        if (!kv.key || cpu_or_memory(kv.key)) continue;
        const uint32_t r = res_id(c, kv.key);
        if (std::any_of(out.begin(), out.end(), [r](const ExtQty& e) { return e.res == r; })) continue;
        int64_t v = 0;
        const uint8_t err = parse_quantity(kv.val, 0, &v) != KS_OK ? EXT_PARSE : EXT_OK;
        out.push_back({r, err, err ? 0 : v});
    }
    return out;
}

// append a bound pod; a tracked key that is already present REPLACES its row (last one wins, as a map would): the old
// row is removed so its requests are no longer charged, and the device copy is re-uploaded from the host truth
static void bound_push(ksh_context* c, const ks_pod_obj* pod, uint64_t h, size_t lns, size_t lname, int32_t node, int64_t cpu,
                       int64_t mem) {
    const bool tracked = lns + lname > 0; // a pod without namespace and name cannot be addressed by later events
    int32_t prio = 0;
    if (tracked) {
        const int64_t old = btab_find_slot(c, h, pod, lns, lname);
        if (old >= 0) {
            const size_t old_pos = slot_low(c->btab.slots[(size_t)old]) - 2;
            prio = c->bprio[old_pos]; // the same pod: spec.priority is immutable
            bound_erase(c, old_pos);
            c->dirty = true;
        }
    }
    const size_t pos = c->bnode.size();
    c->bext.push_back(pod_ext(c, pod));
    c->bnode.push_back(node);
    c->bcpu.push_back(cpu);
    c->bmem.push_back(mem);
    c->bprio.push_back(prio);
    c->bhash.push_back(tracked ? h : 0);
    c->boff.push_back(c->bkeys.size());
    c->blen.push_back(tracked ? (uint32_t)(lns + 1 + lname) : 0);
    if (!tracked) return;
    c->live_key_bytes += lns + 1 + lname;
    c->bkeys.insert(c->bkeys.end(), nz(pod->ns), nz(pod->ns) + lns);
    c->bkeys.push_back('/');
    c->bkeys.insert(c->bkeys.end(), nz(pod->name), nz(pod->name) + lname);
    if ((c->btab.used + 1) * 2 > c->btab.slots.size()) { // also the first insertion
        btab_rebuild(c, c->bnode.size());                // places every row, the new one included
        return;
    }
    // one probe walk: an older row with the same key is re-pointed; else the first free slot on the way is taken
    const size_t mask = c->btab.slots.size() - 1;
    int64_t free_slot = -1;
    for (size_t i = h & mask;; i = (i + 1) & mask) {
        const uint64_t s = c->btab.slots[i];
        if (s == 0) {
            if (free_slot < 0) {
                free_slot = (int64_t)i;
                c->btab.used++;
            }
            break;
        }
        if (slot_low(s) == 1) {
            if (free_slot < 0) free_slot = (int64_t)i;
        } else if ((s >> 32) == (h >> 32) && bkey_equal(c, slot_low(s) - 2, h, pod, lns, lname)) {
            c->btab.slots[i] = btab_word(h, pos);
            return;
        }
    }
    c->btab.slots[(size_t)free_slot] = btab_word(h, pos);
}

// bound_push for a pod whose key is not hashed yet
static void bound_push(ksh_context* c, const ks_pod_obj* pod, int32_t node, int64_t cpu, int64_t mem) {
    size_t lns, lname;
    const uint64_t h = pod_key_hash(pod, &lns, &lname);
    bound_push(c, pod, h, lns, lname, node, cpu, mem);
}

static void bound_erase(ksh_context* c, size_t pos) { // swap-remove
    const size_t last = c->bnode.size() - 1;
    c->live_key_bytes -= c->blen[pos];
    if (c->blen[pos]) {
        const int64_t i = btab_slot_of_pos(c, pos);
        if (i >= 0) c->btab.slots[(size_t)i] = 1; // tombstone
    }
    if (pos != last) {
        if (c->blen[last]) {
            const int64_t i = btab_slot_of_pos(c, last);
            if (i >= 0) c->btab.slots[(size_t)i] = btab_word(c->bhash[last], pos);
        }
        c->bnode[pos] = c->bnode[last];
        c->bcpu[pos] = c->bcpu[last];
        c->bmem[pos] = c->bmem[last];
        c->bhash[pos] = c->bhash[last];
        c->boff[pos] = c->boff[last];
        c->blen[pos] = c->blen[last];
        c->bprio[pos] = c->bprio[last];
        c->bext[pos] = std::move(c->bext[last]);
    }
    c->bext.pop_back();
    c->bnode.pop_back();
    c->bcpu.pop_back();
    c->bmem.pop_back();
    c->bhash.pop_back();
    c->boff.pop_back();
    c->blen.pop_back();
    c->bprio.pop_back();
    if (c->bnode.empty()) c->bkeys.clear(); // otherwise erased keys wait for gc_bound_keys
}

static void bound_clear(ksh_context* c) {
    c->bext.clear();
    c->bnode.clear();
    c->bcpu.clear();
    c->bmem.clear();
    c->bhash.clear();
    c->boff.clear();
    c->blen.clear();
    c->bprio.clear();
    c->bkeys.clear();
    c->btab.clear();
    c->live_key_bytes = 0;
}

static const char* const NO_SNAPSHOT =
    "packing-only context (KSH_DEVICE_NONE): no device snapshot, nothing is computed on the host";

static int upload(ksh_context* c) {
    if (!c->snap) return fail(KS_ERR_NO_DEVICE, NO_SNAPSHOT);
    if (!c->dirty) return KS_OK;
    std::vector<uint64_t> lab((size_t)c->N * c->W, 0);
    fill_label_words(c, lab.data());
    int rc = ks_snapshot_set_nodes(c->snap, c->N, c->W, c->alloc_cpu.data(), c->alloc_mem.data(), lab.data());
    if (rc) return rc;
    rc = ks_snapshot_set_bound(c->snap, c->bnode.size(), c->bnode.data(), c->bcpu.data(), c->bmem.data());
    if (rc) return rc;
    c->dirty = false;
    return KS_OK;
}

static inline int32_t node_index_of(const ksh_context* c, const char* name) {
    const int64_t id = c->names.find(nz(name), '\0', "");
    return id < 0 ? -1 : c->nameid2idx[(size_t)id];
}

// ---- packing a batch of pending pods (src/util.rs:54-75 + the selector side of src/predicates.rs:45-61) ----
// One pass over the objects does all the string work: request totals (quantity parse) and ONE interner lookup per selector
// entry, whose pair ids are parked per thread in array order.  Then the dictionary grows (serial, tiny), and a second pass over
// the same ranges turns the parked pair ids into selector bits without touching a string again.  Every selector pair of the
// batch that some node carries gets a dictionary bit, first occurrence (in pod order) first, whatever the thread count.
constexpr uint64_t PACK_MIN_PER_THREAD = 2048; // both passes must cut [0,n) into the same ranges

struct PackScratch {
    std::vector<std::vector<int32_t>> pids;  // per thread: pair id (-1 = unknown pair) of every selector entry of its range, in order
    std::vector<std::vector<uint32_t>> need; // per thread: known pairs some node carries that have no dictionary bit yet
};

static int pack_scan(const ksh_context* c, const ks_pod_obj* pods, uint64_t n, int64_t* req_cpu, int64_t* req_mem, PackScratch& ps) {
    ps.pids.assign(host_threads(), {});
    ps.need.assign(host_threads(), {});
    std::vector<RangeError> errs(host_threads());
    parallel_ranges(n, PACK_MIN_PER_THREAD, [&](unsigned t, uint64_t b, uint64_t e) {
        std::vector<int32_t>& pids = ps.pids[t];
        std::vector<uint32_t>& need = ps.need[t];
        for (uint64_t p = b; p < e; p++) {
            const ks_pod_obj& pod = pods[p];
            const int rc = total_pod_resources(&pod, &req_cpu[p], &req_mem[p], &errs[t].msg);
            if (rc) {
                errs[t].rc = rc;
                return;
            }
            if (!(pod.has_spec && pod.has_node_selector)) continue;
            for (uint32_t i = 0; i < pod.n_selector; i++) {
                const int64_t pid = c->pairs.find(nz(pod.selector[i].key), '\0', nz(pod.selector[i].val));
                pids.push_back((int32_t)pid);
                if (pid < 0 || c->pair_bit[(size_t)pid] >= 0 || c->pair_refcnt[(size_t)pid] == 0) continue; // unknown pair, known bit, or absent everywhere
                if (need.empty() || need.back() != (uint32_t)pid) need.push_back((uint32_t)pid);
            }
        }
    });
    return first_error(errs);
}

static int grow_dictionary(ksh_context* c, const PackScratch& ps, const ks_pod_obj* pods, uint64_t n) {
    const std::vector<std::vector<uint32_t>>& need = ps.need;
    // Room check first.  The dictionary only has to cover the pairs THIS batch names (node columns are re-uploaded
    // whenever it changes), so when the pairs accumulated over the context's lifetime leave no room - e.g. hostname
    // selectors across more than 511 nodes over time - it is rebuilt from the current batch instead of failing.
    {
        std::vector<uint32_t> fresh;
        std::vector<uint8_t> seen(c->pairs.size(), 0);
        for (const auto& v : need)
            for (uint32_t pid : v)
                if (!seen[pid]) {
                    seen[pid] = 1;
                    fresh.push_back(pid);
                }
        if (words_for_bits((uint32_t)(c->bit2pair.size() + fresh.size())) > KS_MAX_LABEL_WORDS) {
            compact_dictionary(c);
            if (words_for_bits((uint32_t)(c->bit2pair.size() + fresh.size())) > KS_MAX_LABEL_WORDS) {
                for (uint32_t pid : c->bit2pair) c->pair_bit[pid] = -1;
                c->bit2pair.clear();
                c->dirty = true;
                std::fill(seen.begin(), seen.end(), 0);
                for (uint64_t p = 0; p < n; p++) { // rare path: serial re-scan, every live pair of the batch
                    const ks_pod_obj& pod = pods[p];
                    if (!(pod.has_spec && pod.has_node_selector)) continue;
                    for (uint32_t i = 0; i < pod.n_selector; i++) {
                        const int64_t pid = c->pairs.find(nz(pod.selector[i].key), '\0', nz(pod.selector[i].val));
                        if (pid < 0 || c->pair_refcnt[(size_t)pid] == 0 || seen[(size_t)pid]) continue;
                        seen[(size_t)pid] = 1;
                        if (words_for_bits((uint32_t)c->bit2pair.size() + 1) > KS_MAX_LABEL_WORDS)
                            return fail(KS_ERR_RANGE, "one batch names more than 511 distinct (key,value) pairs that nodes carry: split the batch");
                        c->pair_bit[(size_t)pid] = (int32_t)c->bit2pair.size();
                        c->bit2pair.push_back((uint32_t)pid);
                    }
                }
                update_words(c);
                return KS_OK;
            }
        }
    }
    for (const auto& v : need)
        for (uint32_t pid : v) {
            const int rc = assign_bit(c, pid);
            if (rc) return rc;
        }
    update_words(c);
    return KS_OK;
}

// selector words of the batch under the current dictionary, from the pair ids parked by pack_scan (same ranges, same order)
static void pack_selectors(const ksh_context* c, const ks_pod_obj* pods, uint64_t n, const PackScratch& ps, uint64_t* sel,
                           uint32_t stride) {
    const uint32_t absent = c->W * 64 - 1;
    parallel_ranges(n, PACK_MIN_PER_THREAD, [&](unsigned t, uint64_t b, uint64_t e) {
        const int32_t* pid = ps.pids[t].data();
        for (uint64_t p = b; p < e; p++) {
            uint64_t* row = sel + p * stride;
            for (uint32_t w = 0; w < stride; w++) row[w] = 0;
            if (!(pods[p].has_spec && pods[p].has_node_selector)) continue;
            for (uint32_t i = 0; i < pods[p].n_selector; i++) {
                const int32_t id = *pid++;
                const int32_t b_ = id < 0 ? -1 : c->pair_bit[(size_t)id];
                const uint32_t bit = b_ < 0 ? absent : (uint32_t)b_; // a pair no node carries: never-set bit
                row[bit >> 6] |= 1ull << (bit & 63);
            }
        }
    });
}

// ---- calls that need the device ----
// Each such call makes this check where it first needs the device: a packing-only context has no snapshot, and a library built
// with a device stand-in (tests/native) may lack the optional entry.
template <class F>
static int device_ready(const ksh_context* c, F* entry, const char* name) {
    if (!c->snap) return fail(KS_ERR_NO_DEVICE, NO_SNAPSHOT);
    if (!entry) return fail(KS_ERR_NO_DEVICE, std::string("this library has no ") + name);
    return KS_OK;
}

// Packs a batch into the context's pk_* set (kept between calls: fresh pages cost more than the packing), uploads the snapshot,
// and describes the packed batch in *kp.  *kp stays valid until the next pack; the context lock held for the whole call keeps it so.
static int pack_batch(ksh_context* c, const ks_pod_obj* pods, uint64_t n, ks_pods* kp) {
    c->pk_cpu.resize(n);
    c->pk_mem.resize(n);
    PackScratch ps;
    int rc = pack_scan(c, pods, n, c->pk_cpu.data(), c->pk_mem.data(), ps);
    if (rc) return rc;
    rc = grow_dictionary(c, ps, pods, n);
    if (rc) return rc;
    c->pk_sel.resize((size_t)n * c->W);
    pack_selectors(c, pods, n, ps, c->pk_sel.data(), c->W);
    *kp = ks_pods{n, c->pk_cpu.data(), c->pk_mem.data(), c->pk_sel.data(), KS_MEM_HOST};
    return upload(c);
}

// A string-list output: entries back to back in buf[0, cap), each NUL-terminated.  An entry that does not fit is skipped (offset -1),
// and a later, shorter entry may still fit.
struct StringList {
    char* buf;
    size_t cap;
    size_t used = 0;
    // s[0, len) holds the entry with its terminating NUL(s); returns its offset, or -1 if it does not fit
    int64_t append(const char* s, size_t len) {
        if (used + len > cap) return -1;
        std::memcpy(buf + used, s, len);
        used += len;
        return (int64_t)(used - len);
    }
};

extern "C" {

int ksh_parse_cpu_millicores(const char* q, int64_t* out) try {
    if (!out) return fail(KS_ERR_INVALID, "out is NULL");
    std::string err;
    const int rc = parse_cpu(q, out, &err);
    return rc ? fail(rc, err) : KS_OK;
}
KSH_CATCH

int ksh_parse_memory_bytes(const char* q, int64_t* out) try {
    if (!out) return fail(KS_ERR_INVALID, "out is NULL");
    std::string err;
    const int rc = parse_mem(q, out, &err);
    return rc ? fail(rc, err) : KS_OK;
}
KSH_CATCH

int ksh_total_pod_resources(const ks_pod_obj* pod, int64_t* cpu, int64_t* mem) try {
    if (!pod || !cpu || !mem) return fail(KS_ERR_INVALID, "NULL argument");
    std::string err;
    const int rc = total_pod_resources(pod, cpu, mem, &err);
    return rc ? fail(rc, err) : KS_OK;
}
KSH_CATCH

int ksh_is_pod_bound(const ks_pod_obj* pod) { return pod && pod->has_spec && pod->node_name != nullptr; } // util.rs:38-45

int ksh_context_create(int device, ksh_context** out) try {
    if (!out) return fail(KS_ERR_INVALID, "out is NULL");
    *out = nullptr;
    ksh_context* c = new (std::nothrow) ksh_context();
    if (!c) return fail(KS_ERR_NOMEM, "out of host memory");
    if (device != KSH_DEVICE_NONE) { // KSH_DEVICE_NONE: packer only, every call that needs the device fails
        int rc = ks_snapshot_create(device, &c->snap);
        if (rc) {
            delete c;
            return rc;
        }
    }
    *out = c;
    return KS_OK;
}
KSH_CATCH

void ksh_context_destroy(ksh_context* c) {
    if (!c) return;
    ks_snapshot_destroy(c->snap);
    delete c;
}

uint32_t ksh_context_num_nodes(const ksh_context* c) {
    if (!c) return 0;
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    return c->N;
}
uint32_t ksh_context_label_words(const ksh_context* c) {
    if (!c) return 0;
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    return c->W;
}
uint64_t ksh_context_num_bound(const ksh_context* c) {
    if (!c) return 0;
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    return c->bnode.size();
}

int ksh_context_export_packed(const ksh_context* c, int64_t* alloc_cpu, int64_t* alloc_mem, uint64_t* labels,
                              int32_t* bound_node, int64_t* bound_cpu, int64_t* bound_mem) try {
    if (!c) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    if (c->N && (!alloc_cpu || !alloc_mem || !labels)) return fail(KS_ERR_INVALID, "NULL node array");
    if (!c->bnode.empty() && (!bound_node || !bound_cpu || !bound_mem)) return fail(KS_ERR_INVALID, "NULL bound array");
    if (c->N) {
        std::memcpy(alloc_cpu, c->alloc_cpu.data(), (size_t)c->N * 8);
        std::memcpy(alloc_mem, c->alloc_mem.data(), (size_t)c->N * 8);
        fill_label_words(c, labels);
    }
    if (!c->bnode.empty()) {
        std::memcpy(bound_node, c->bnode.data(), c->bnode.size() * 4);
        std::memcpy(bound_cpu, c->bcpu.data(), c->bcpu.size() * 8);
        std::memcpy(bound_mem, c->bmem.data(), c->bmem.size() * 8);
    }
    return KS_OK;
}
KSH_CATCH

ks_snapshot* ksh_context_snapshot(ksh_context* c) {
    if (!c) return nullptr;
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    if (upload(c)) return nullptr;
    return c->snap;
}

int ksh_context_set_nodes(ksh_context* c, const ks_node_obj* nodes, uint32_t n) try {
    if (!c || (n && !nodes)) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    // validate first (quantities parsed by all host threads), then replace
    std::vector<int64_t> ac(n), am(n);
    std::vector<RangeError> errs(host_threads());
    parallel_ranges(n, 2048, [&](unsigned t, uint64_t b, uint64_t e) {
        for (uint64_t i = b; i < e; i++) {
            const int rc = parse_node_allocatable(nodes[i], &ac[i], &am[i], &errs[t].msg);
            if (rc) {
                errs[t].rc = rc;
                return;
            }
        }
    });
    int rc = first_error(errs);
    if (rc) return rc;
    // selector pairs that already have a bit keep it if some new node still carries the pair
    std::vector<std::string> named; // "key\0value" of the dictionary, in bit order
    named.reserve(c->bit2pair.size());
    for (uint32_t pid : c->bit2pair) named.emplace_back(c->pairs.str(pid), c->pairs.ents[pid].len);
    c->names.clear();
    c->nameid2idx.clear();
    c->idx2nameid.assign(n, 0);
    c->pairs.clear();
    c->live_pairs = 0;
    c->pair_refcnt.clear();
    c->pair_bit.clear();
    c->bit2pair.clear();
    c->node_pids.assign(n, {});
    c->node_ext.assign(n, {});
    c->N = n;
    c->alloc_cpu.swap(ac);
    c->alloc_mem.swap(am);
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t id = c->names.intern(nz(nodes[i].name), '\0', "");
        if (id == c->nameid2idx.size()) c->nameid2idx.push_back((int32_t)i); // first node of a name wins
        c->idx2nameid[i] = id;
        node_pairs_set(c, i, nodes[i]);
        c->node_ext[i] = node_ext(c, nodes[i]);
    }
    for (const std::string& pk : named) {
        const char* k = pk.c_str();
        const char* v = k + std::strlen(k) + 1;
        const int64_t pid = c->pairs.find(k, '\0', v);
        if (pid >= 0 && c->pair_refcnt[(size_t)pid] > 0) {
            c->pair_bit[(size_t)pid] = (int32_t)c->bit2pair.size();
            c->bit2pair.push_back((uint32_t)pid);
        }
    }
    c->W = words_for_bits((uint32_t)c->bit2pair.size());
    bound_clear(c);
    c->taints.clear();
    c->dirty = true;
    return KS_OK;
}
KSH_CATCH

int ksh_context_upsert_node(ksh_context* c, const ks_node_obj* node, uint32_t* out_idx) try {
    if (!c || !node) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    int64_t ac, am;
    std::string err;
    const int rc = parse_node_allocatable(*node, &ac, &am, &err);
    if (rc) return fail(rc, err);
    const uint32_t id = c->names.intern(nz(node->name), '\0', "");
    if (id == c->nameid2idx.size()) c->nameid2idx.push_back(-1);
    uint32_t idx;
    if (c->nameid2idx[id] < 0) { // new node (or one that had been removed): appended
        idx = c->N++;
        c->nameid2idx[id] = (int32_t)idx;
        c->idx2nameid.push_back(id);
        c->alloc_cpu.push_back(ac);
        c->alloc_mem.push_back(am);
        c->node_pids.emplace_back();
        c->node_ext.emplace_back();
    } else {
        idx = (uint32_t)c->nameid2idx[id];
        c->alloc_cpu[idx] = ac;
        c->alloc_mem[idx] = am;
        node_pairs_release(c, idx);
    }
    node_pairs_set(c, idx, *node);
    c->node_ext[idx] = node_ext(c, *node);
    gc_pairs(c);
    c->dirty = true;
    if (out_idx) *out_idx = idx;
    return KS_OK;
}
KSH_CATCH

int ksh_context_remove_node(ksh_context* c, const char* name) try {
    if (!c || !name) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    const int32_t found = node_index_of(c, name);
    if (found < 0) return KS_OK;
    const uint32_t idx = (uint32_t)found;
    c->taints.erase(name);
    node_pairs_release(c, idx);
    c->nameid2idx[c->idx2nameid[idx]] = -1;
    c->idx2nameid.erase(c->idx2nameid.begin() + idx);
    c->alloc_cpu.erase(c->alloc_cpu.begin() + idx);
    c->alloc_mem.erase(c->alloc_mem.begin() + idx);
    c->node_pids.erase(c->node_pids.begin() + idx);
    c->node_ext.erase(c->node_ext.begin() + idx);
    c->N--;
    // later nodes move down by one index; a name carried by several rows points to its first remaining row
    for (uint32_t i = c->N; i-- > idx;) c->nameid2idx[c->idx2nameid[i]] = (int32_t)i;
    for (uint32_t i = 0; i < idx; i++)
        if (c->nameid2idx[c->idx2nameid[i]] > (int32_t)i) c->nameid2idx[c->idx2nameid[i]] = (int32_t)i;
    // pods bound to the removed node disappear from every later LIST; indices above it move down
    for (size_t p = 0; p < c->bnode.size();) {
        if ((uint32_t)c->bnode[p] == idx) {
            bound_erase(c, p);
        } else {
            if ((uint32_t)c->bnode[p] > idx) c->bnode[p]--;
            p++;
        }
    }
    gc_pairs(c);
    gc_names(c);
    gc_bound_keys(c);
    c->dirty = true;
    return KS_OK;
}
KSH_CATCH

int ksh_context_pod_bound(ksh_context* c, const ks_pod_obj* pod) try {
    if (!c || !pod) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    if (!ksh_is_pod_bound(pod)) return KS_OK;
    const int32_t node = node_index_of(c, pod->node_name);
    if (node < 0) return KS_OK;
    int64_t cpu, mem;
    std::string err;
    const int rc = total_pod_resources(pod, &cpu, &mem, &err);
    if (rc) return fail(rc, err);
    bound_push(c, pod, node, cpu, mem); // an update of a pod already known replaces its row
    gc_bound_keys(c);
    c->dirty = true;
    return KS_OK;
}
KSH_CATCH

int ksh_context_pod_deleted(ksh_context* c, const ks_pod_obj* pod) try {
    if (!c || !pod) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    size_t lns, lname;
    const uint64_t h = pod_key_hash(pod, &lns, &lname);
    if (lns + lname == 0) return KS_OK;
    const int64_t slot = btab_find_slot(c, h, pod, lns, lname);
    if (slot < 0) return KS_OK;
    bound_erase(c, slot_low(c->btab.slots[(size_t)slot]) - 2);
    gc_bound_keys(c);
    c->dirty = true;
    return KS_OK;
}
KSH_CATCH

const char* ksh_context_node_name(const ksh_context* c, uint32_t idx) {
    if (!c) return nullptr;
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    return idx < c->N ? c->names.str(c->idx2nameid[idx]) : nullptr;
}

int ksh_context_set_cluster_pods(ksh_context* c, const ks_pod_obj* pods, uint64_t n) try {
    if (!c || (n && !pods)) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    if (n > 0xFFFFFFF0ull) return fail(KS_ERR_RANGE, "too many pods");
    // validate first, then replace.  Per pod (all host threads): spec.nodeName -> node index (the field selector of
    // predicates.rs:22-25), request totals (predicates.rs:37), key hash.
    std::vector<int32_t>& node = c->tmp_node;
    std::vector<int64_t>&cpus = c->tmp_cpu, &mems = c->tmp_mem;
    std::vector<uint64_t>& hashes = c->tmp_hash;
    std::vector<uint32_t>& lens = c->tmp_len;
    node.resize(n);
    cpus.resize(n);
    mems.resize(n);
    hashes.resize(n);
    lens.resize(2 * n);
    std::vector<RangeError> errs(host_threads());
    parallel_ranges(n, 4096, [&](unsigned t, uint64_t b, uint64_t e) {
        for (uint64_t p = b; p < e; p++) {
            node[p] = ksh_is_pod_bound(&pods[p]) ? node_index_of(c, pods[p].node_name) : -1;
            if (node[p] < 0) continue;
            const int rc = total_pod_resources(&pods[p], &cpus[p], &mems[p], &errs[t].msg);
            if (rc) {
                errs[t].rc = rc;
                return;
            }
            size_t lns, lname;
            hashes[p] = pod_key_hash(&pods[p], &lns, &lname);
            lens[2 * p] = (uint32_t)lns;
            lens[2 * p + 1] = (uint32_t)lname;
        }
    });
    const int rc = first_error(errs);
    if (rc) return rc;
    bound_clear(c);
    uint64_t kept = 0, key_bytes = 0;
    for (uint64_t p = 0; p < n; p++)
        if (node[p] >= 0) {
            kept++;
            key_bytes += (uint64_t)lens[2 * p] + lens[2 * p + 1] + 1;
        }
    c->bnode.reserve(kept);
    c->bcpu.reserve(kept);
    c->bmem.reserve(kept);
    c->bhash.reserve(kept);
    c->boff.reserve(kept);
    c->blen.reserve(kept);
    c->bprio.reserve(kept);
    c->bext.reserve(kept);
    c->bkeys.reserve(key_bytes);
    btab_rebuild(c, kept); // sized once for the whole list
    for (uint64_t p = 0; p < n; p++)
        if (node[p] >= 0) bound_push(c, &pods[p], hashes[p], lens[2 * p], lens[2 * p + 1], node[p], cpus[p], mems[p]);
    c->dirty = true;
    return KS_OK;
}
KSH_CATCH

int ksh_pack_pods(ksh_context* c, const ks_pod_obj* pods, uint64_t n, int64_t* req_cpu, int64_t* req_mem,
                  uint64_t* sel, uint32_t stride) try {
    if (!c || (n && (!pods || !req_cpu || !req_mem || !sel))) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    PackScratch ps;
    int rc = pack_scan(c, pods, n, req_cpu, req_mem, ps);
    if (rc) return rc;
    rc = grow_dictionary(c, ps, pods, n);
    if (rc) return rc;
    if (stride < c->W) return fail(KS_ERR_INVALID, "sel_stride_words smaller than the dictionary's word count");
    pack_selectors(c, pods, n, ps, sel, stride);
    return (int)c->W;
}
KSH_CATCH

int ksh_check_node_validity(ksh_context* c, const ks_pod_obj* pod, uint32_t node_idx) try {
    if (!c || !pod) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    if (node_idx >= c->N) return fail(KS_ERR_INVALID, "node index out of range");
    ks_pods kp;
    const int rc = pack_batch(c, pod, 1, &kp);
    if (rc) return rc;
    return ks_check_cell(c->snap, kp.req_cpu[0], kp.req_mem[0], kp.sel, node_idx);
}
KSH_CATCH

int ksh_select_nodes(ksh_context* c, const ks_pod_obj* pods, uint64_t n, int policy, int32_t* out_node_idx,
                     int64_t* out_score, uint32_t* out_cnt) try {
    if (!c || (n && !pods)) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    if (n == 0) return KS_OK;
    ks_pods kp;
    const int rc = pack_batch(c, pods, n, &kp);
    if (rc) return rc;
    ks_bindings kb{out_node_idx, out_score, out_cnt, KS_MEM_HOST, nullptr, 0, KS_MEM_HOST, nullptr, nullptr};
    return ks_select(c->snap, &kp, policy, KS_SELECT_AUTO, &kb, nullptr);
}
KSH_CATCH

int ksh_rank_nodes(ksh_context* c, const ks_pod_obj* pods, uint64_t n, int policy, uint32_t k, int32_t* out_node_idx,
                   int64_t* out_score, uint32_t* out_cnt) try {
    if (!c || (n && !pods)) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    int rc = device_ready(c, ks_select_topk, "ks_select_topk");
    if (rc) return rc;
    if (k == 0 || k > KS_TOPK_MAX) return fail(KS_ERR_RANGE, "k must be in [1, " + std::to_string(KS_TOPK_MAX) + "]");
    if (n == 0) return KS_OK;
    if (!out_node_idx) return fail(KS_ERR_INVALID, "out_node_idx is NULL");
    ks_pods kp;
    rc = pack_batch(c, pods, n, &kp);
    if (rc) return rc;
    return ks_select_topk(c->snap, &kp, policy, k, out_node_idx, out_score, out_cnt, KS_MEM_HOST, nullptr);
}
KSH_CATCH

int ksh_select_node_for_pod(ksh_context* c, const ks_pod_obj* pods, uint64_t n, uint32_t attempts, uint64_t seed,
                            uint64_t first_pod_index, int32_t* out_node_idx, uint32_t* out_attempts,
                            int32_t* out_draw_node, uint8_t* out_draw_code) try {
    if (!c || (n && !pods)) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    if (n == 0) return KS_OK;
    ks_pods kp;
    const int rc = pack_batch(c, pods, n, &kp);
    if (rc) return rc;
    return ks_select_sampling(c->snap, &kp, attempts, seed, first_pod_index, out_node_idx, out_attempts, out_draw_node,
                              out_draw_code);
}
KSH_CATCH

// A pod that comes back to reconcile() unbound although this context bound it earlier (the caller's POST failed or
// raced, error_policy requeued it - src/main.rs:105-108,122-125): the reference's next LIST would not show it, so
// the earlier charge is dropped before the new selection.  Returns true if a row was released.
static bool release_earlier_binding(ksh_context* c, const ks_pod_obj* pod) {
    size_t lns, lname;
    const uint64_t h = pod_key_hash(pod, &lns, &lname);
    if (lns + lname == 0) return false;
    const int64_t slot = btab_find_slot(c, h, pod, lns, lname);
    if (slot < 0) return false;
    bound_erase(c, slot_low(c->btab.slots[(size_t)slot]) - 2);
    c->dirty = true; // the device's free[] still carries the old charge: re-upload before the next evaluation
    return true;
}

// corev1::Binding{metadata, target: ObjectReference{name}}  (src/main.rs:83-91), the body of
// POST /api/v1/namespaces/{ns}/pods/{name}/binding
static std::string binding_body(const ksh_context* c, const ks_pod_obj* pod, uint32_t node_idx) {
    std::string s = "{\"apiVersion\":\"v1\",\"kind\":\"Binding\",\"metadata\":";
    if (pod->metadata_json && pod->metadata_json[0]) { // src/main.rs:88: metadata: pod.metadata.clone()
        s += pod->metadata_json;
    } else {
        s += "{\"name\":\"";
        json_escape(s, pod->name);
        s += "\",\"namespace\":\"";
        json_escape(s, pod->ns);
        s += "\"}";
    }
    s += ",\"target\":{\"name\":\"";
    json_escape(s, ksh_context_node_name(c, node_idx));
    s += "\"}}";
    return s;
}

int ksh_reconcile(ksh_context* c, const ks_pod_obj* pod, int policy, int32_t* node_idx, char* json, size_t cap) try {
    if (!c || !pod || !node_idx) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    *node_idx = -1;
    if (json && cap) json[0] = '\0';
    if (ksh_is_pod_bound(pod)) return KSH_RECONCILE_OK; // src/main.rs:74-76
    release_earlier_binding(c, pod);
    int32_t idx = -1;
    int rc = ksh_select_nodes(c, pod, 1, policy, &idx, nullptr, nullptr); // src/main.rs:78
    if (rc) return rc;
    if (idx < 0) return KSH_RECONCILE_NO_NODE_FOUND; // src/main.rs:116-118
    if (!pod->ns || !pod->name) {
        fail(KS_ERR_INVALID, "pod has no namespace/name (reference: unwrap panic, src/main.rs:80)");
        return KSH_RECONCILE_BINDING_OBJECT_FAILED;
    }
    int64_t cpu, mem;
    rc = ksh_total_pod_resources(pod, &cpu, &mem);
    if (rc) return rc;
    // what the next LIST would report once the binding is accepted (src/predicates.rs:34 after src/main.rs:103)
    rc = ks_snapshot_apply_bind(c->snap, idx, cpu, mem);
    if (rc) {
        c->dirty = true; // the device may or may not carry the bind: re-upload from the host truth next time
        return rc;
    }
    bound_push(c, pod, idx, cpu, mem);
    *node_idx = idx;
    if (json && cap) std::snprintf(json, cap, "%s", binding_body(c, pod, (uint32_t)idx).c_str());
    return KSH_RECONCILE_OK;
}
KSH_CATCH

// reconcile()'s outcome for a pod of a batch before the device: a bound pod is done (src/main.rs:74-76), a pod without namespace
// or name cannot get a Binding (reference: unwrap panic, src/main.rs:80), and any other goes to the device and stays
// NO_NODE_FOUND until it binds (src/main.rs:116-118), with an earlier binding of it by this context dropped first.
static int32_t reconcile_status(ksh_context* c, const ks_pod_obj* pod) {
    if (ksh_is_pod_bound(pod)) return KSH_RECONCILE_OK;
    if (!pod->ns || !pod->name) return KSH_RECONCILE_BINDING_OBJECT_FAILED;
    release_earlier_binding(c, pod);
    return KSH_RECONCILE_NO_NODE_FOUND;
}

// The host side of a bind the device committed: the row the next LIST would show, the pod's status and node, and its Binding
// body in the string list (when body_off is given).
static void commit_bind(ksh_context* c, const ks_pod_obj* pod, int32_t node, int64_t cpu, int64_t mem, int32_t* status,
                        int32_t* node_idx, StringList& bodies, int64_t* body_off) {
    bound_push(c, pod, node, cpu, mem);
    *status = KSH_RECONCILE_OK;
    *node_idx = node;
    if (body_off) {
        const std::string body = binding_body(c, pod, (uint32_t)node);
        *body_off = bodies.append(body.c_str(), body.size() + 1);
    }
}

// reconcile() for a drained queue: one pack, one micro-batch loop on the device (select -> claims resolved in array order ->
// losers re-selected against what is left), then the host-side commit of every bind (what the next LIST would show)
int ksh_reconcile_batch(ksh_context* c, const ks_pod_obj* pods, uint64_t n, int policy, int32_t* out_status, int32_t* out_node_idx,
                        char* json, size_t cap, int64_t* out_json_off, uint32_t* out_rounds) try {
    if (!c || (n && (!pods || !out_status || !out_node_idx))) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    if (out_rounds) *out_rounds = 0;
    std::vector<uint64_t> todo;
    std::vector<ks_pod_obj> sub; // shallow copies: the pods that actually go to the device, in arrival order
    for (uint64_t i = 0; i < n; i++) {
        out_node_idx[i] = -1;
        if (out_json_off) out_json_off[i] = -1;
        out_status[i] = reconcile_status(c, &pods[i]);
        if (out_status[i] != KSH_RECONCILE_NO_NODE_FOUND) continue;
        todo.push_back(i);
        sub.push_back(pods[i]);
    }
    if (todo.empty()) return KS_OK;
    ks_pods kp;
    int rc = pack_batch(c, sub.data(), sub.size(), &kp);
    if (rc) return rc;
    std::vector<int32_t> idx(sub.size(), -1);
    rc = ks_stream_bind(c->snap, &kp, policy, idx.data(), nullptr, out_rounds); // commits capacity on the device
    if (rc) {
        c->dirty = true; // some rounds may have committed claims on the device: the host list is the truth
        return rc;
    }
    StringList bodies{json, cap};
    for (size_t k = 0; k < todo.size(); k++) {
        const uint64_t i = todo[k];
        if (idx[k] >= 0)
            commit_bind(c, &pods[i], idx[k], kp.req_cpu[k], kp.req_mem[k], &out_status[i], &out_node_idx[i], bodies,
                        json && out_json_off ? &out_json_off[i] : nullptr);
    }
    return KS_OK;
}
KSH_CATCH

// A cut of n pods into n_cut groups or gangs (`what`) by offset: each of 1 to max_size pods (no limit at UINT64_MAX) and
// its min_member within its size
static int check_cut(const std::string& what, const uint64_t* offset, uint64_t n_cut, const uint32_t* min_member,
                     uint64_t n, uint64_t max_size) {
    if (offset[0] != 0) return fail(KS_ERR_INVALID, what + "_offset[0] must be 0");
    for (uint64_t j = 0; j < n_cut; j++) {
        if (offset[j + 1] < offset[j]) return fail(KS_ERR_INVALID, what + " offsets decrease");
        const uint64_t size = offset[j + 1] - offset[j];
        if (size == 0 || size > max_size)
            return fail(KS_ERR_RANGE, max_size == UINT64_MAX ? "a " + what + " has no pod"
                                                             : "a " + what + " has " + std::to_string(size) + " pods (1.." +
                                                                   std::to_string(max_size) + ")");
        if (min_member[j] > size) return fail(KS_ERR_RANGE, "min_member above the " + what + "'s size");
    }
    if (offset[n_cut] != n) return fail(KS_ERR_INVALID, what + "_offset[n_" + what + "s] must be n_pods");
    return KS_OK;
}

// reconcile() for pod groups: ksh_reconcile_batch's filtering, then ks_gang_bind over the pods that go to the device,
// one sub-group per group; already bound members count toward min_member
int ksh_reconcile_gangs(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const uint64_t* group_offset, uint64_t n_groups,
                        const uint32_t* min_member, int policy, int32_t* out_status, int32_t* out_node_idx,
                        uint32_t* out_placed, char* json, size_t cap, int64_t* out_json_off) try {
    if (!c || !group_offset || (n && (!pods || !out_status || !out_node_idx)) || (n_groups && !min_member))
        return fail(KS_ERR_INVALID, "NULL argument");
    int rc = check_cut("group", group_offset, n_groups, min_member, n, KS_GANG_MAX_SIZE);
    if (rc) return rc;
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    rc = device_ready(c, ks_gang_bind, "ks_gang_bind");
    if (rc) return rc;
    std::vector<uint64_t> todo, sub_off{0}, sub_group; // the pods that go to the device; sub-group k is group sub_group[k]
    std::vector<uint32_t> sub_min;
    std::vector<ks_pod_obj> sub;
    if (out_placed)
        for (uint64_t g = 0; g < n_groups; g++) out_placed[g] = 0;
    for (uint64_t g = 0; g < n_groups; g++) {
        uint32_t bound = 0; // running members of the group
        const size_t first = todo.size();
        for (uint64_t i = group_offset[g]; i < group_offset[g + 1]; i++) {
            out_node_idx[i] = -1;
            if (out_json_off) out_json_off[i] = -1;
            out_status[i] = reconcile_status(c, &pods[i]); // an earlier binding is dropped whatever the group does
            if (out_status[i] == KSH_RECONCILE_OK) bound++;
            if (out_status[i] == KSH_RECONCILE_NO_NODE_FOUND) todo.push_back(i);
        }
        const uint32_t need = min_member[g] > bound ? min_member[g] - bound : 0;
        if (todo.size() == first) continue;
        if (need > todo.size() - first) { // too few schedulable members: the group cannot commit, nothing is tried
            for (size_t k = first; k < todo.size(); k++) out_status[todo[k]] = KSH_RECONCILE_GANG_UNSATISFIED;
            todo.resize(first);
            continue;
        }
        for (size_t k = first; k < todo.size(); k++) sub.push_back(pods[todo[k]]);
        sub_off.push_back(todo.size());
        sub_group.push_back(g);
        sub_min.push_back(need);
    }
    if (todo.empty()) return KS_OK;
    ks_pods kp;
    rc = pack_batch(c, sub.data(), sub.size(), &kp);
    if (rc) return rc;
    std::vector<int32_t> idx(sub.size(), -1);
    std::vector<uint32_t> placed(sub_group.size());
    ks_gangs kg{sub_group.size(), sub_off.data(), sub_min.data()};
    rc = ks_gang_bind(c->snap, &kp, &kg, policy, idx.data(), nullptr, placed.data(), nullptr); // commits on the device
    if (rc) {
        c->dirty = true; // the device may carry part of the call: the host list is the truth
        return rc;
    }
    StringList bodies{json, cap};
    for (size_t k = 0; k < sub_group.size(); k++) {
        if (out_placed) out_placed[sub_group[k]] = placed[k];
        const bool commit = placed[k] >= sub_min[k];
        for (uint64_t j = sub_off[k]; j < sub_off[k + 1]; j++) {
            const uint64_t i = todo[j];
            if (!commit)
                out_status[i] = KSH_RECONCILE_GANG_UNSATISFIED;
            else if (idx[j] >= 0) // else NoNodeFound
                commit_bind(c, &pods[i], idx[j], kp.req_cpu[j], kp.req_mem[j], &out_status[i], &out_node_idx[i], bodies,
                            json && out_json_off ? &out_json_off[i] : nullptr);
        }
    }
    return KS_OK;
}
KSH_CATCH

int ksh_format_unschedulable(uint32_t n_nodes, const ks_pod_reasons* r, char* buf, size_t cap) try {
    if (!r || (!buf && cap)) return fail(KS_ERR_INVALID, "NULL argument");
    // upstream's order: the reason strings sorted lexicographically
    const struct {
        uint32_t count;
        const char* text;
    } terms[3] = {{r->insufficient_cpu, "Insufficient cpu"},
                  {r->insufficient_memory, "Insufficient memory"},
                  {r->node_selector_mismatch, "node(s) didn't match Pod's node affinity/selector"}};
    std::string s = "0/" + std::to_string(n_nodes) + " nodes are available";
    const char* sep = ": ";
    for (const auto& t : terms) {
        if (!t.count) continue;
        s += sep;
        s += std::to_string(t.count) + " " + t.text;
        sep = ", ";
    }
    s += ".";
    if (cap) std::snprintf(buf, cap, "%s", s.c_str());
    return (int)s.size();
}
KSH_CATCH

int ksh_explain_pods(ksh_context* c, const ks_pod_obj* pods, uint64_t n, ks_pod_reasons* out, char* messages, size_t cap,
                     int64_t* out_msg_off) try {
    if (!c || (n && (!pods || !out))) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    int rc = device_ready(c, ks_explain, "ks_explain");
    if (rc) return rc;
    if (out_msg_off)
        for (uint64_t i = 0; i < n; i++) out_msg_off[i] = -1;
    if (n == 0) return KS_OK;
    ks_pods kp;
    rc = pack_batch(c, pods, n, &kp);
    if (rc) return rc;
    rc = ks_explain(c->snap, &kp, out, KS_MEM_HOST, nullptr);
    if (rc) return rc;
    if (!messages || !out_msg_off) return KS_OK;
    const uint32_t N = c->N; // what pack_batch just gave the snapshot
    StringList list{messages, cap};
    char msg[256]; // the longest message (three 10-digit counts) is under 200 bytes
    for (uint64_t i = 0; i < n; i++) {
        if ((uint64_t)out[i].not_enough_resources + out[i].node_selector_mismatch < N) continue; // a node is feasible
        const int len = ksh_format_unschedulable(N, &out[i], msg, sizeof(msg));
        out_msg_off[i] = list.append(msg, (size_t)len + 1);
    }
    return KS_OK;
}
KSH_CATCH

int ksh_context_set_pod_priorities(ksh_context* c, const ks_pod_obj* pods, const int32_t* priority, uint64_t n) try {
    if (!c || (n && (!pods || !priority))) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    for (uint64_t i = 0; i < n; i++) {
        size_t lns, lname;
        const uint64_t h = pod_key_hash(&pods[i], &lns, &lname);
        if (lns + lname == 0) continue;
        const int64_t slot = btab_find_slot(c, h, &pods[i], lns, lname);
        if (slot >= 0) c->bprio[slot_low(c->btab.slots[(size_t)slot]) - 2] = priority[i];
    }
    return KS_OK; // the device keeps no priorities: nothing to re-upload
}
KSH_CATCH

int ksh_preempt_pods(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const int32_t* pod_priority, uint32_t max_victims,
                     ks_preemption* out, char* victims, size_t cap, int64_t* out_victim_off) try {
    if (!c || (n && (!pods || !pod_priority || !out))) return fail(KS_ERR_INVALID, "NULL argument");
    if (max_victims == 0 || max_victims > KS_PREEMPT_MAX_VICTIMS)
        return fail(KS_ERR_RANGE, "max_victims must be in [1, " + std::to_string(KS_PREEMPT_MAX_VICTIMS) + "]");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    int rc = device_ready(c, ks_preempt, "ks_preempt");
    if (rc) return rc;
    if (out_victim_off)
        for (uint64_t i = 0; i < n; i++) out_victim_off[i] = -1;
    if (n == 0) return KS_OK;
    ks_pods kp;
    rc = pack_batch(c, pods, n, &kp); // after this the device's free[] comes from the bound rows below
    if (rc) return rc;
    const size_t B = c->bnode.size();
    std::vector<int32_t> prio(B);
    for (size_t b = 0; b < B; b++) prio[b] = c->blen[b] ? c->bprio[b] : INT32_MAX; // anonymous: cannot be evicted
    std::vector<int32_t> vic((size_t)n * max_victims);
    ks_bound_pods kb{B, c->bnode.data(), c->bcpu.data(), c->bmem.data(), prio.data()};
    rc = ks_preempt(c->snap, &kp, pod_priority, &kb, max_victims, out, vic.data(), KS_MEM_HOST, nullptr);
    if (rc) return rc;
    if (!victims || !out_victim_off) return KS_OK;
    StringList list{victims, cap};
    std::string keys;
    for (uint64_t i = 0; i < n; i++) {
        if (out[i].node_idx < 0) continue;
        keys.clear();
        for (uint32_t j = 0; j < out[i].n_victims; j++) { // "namespace/name", NUL-terminated, in visit order
            const size_t b = (size_t)vic[(size_t)i * max_victims + j];
            keys.append(c->bkeys.data() + c->boff[b], c->blen[b]);
            keys.push_back('\0');
        }
        out_victim_off[i] = list.append(keys.data(), keys.size());
    }
    return KS_OK;
}
KSH_CATCH

int ksh_drain_nodes(ksh_context* c, const char* const* node_names, uint64_t n, const ks_pod_obj* pods,
                    const uint64_t* pod_offset, int policy, uint32_t flags, uint32_t* out_placed, int32_t* out_node_idx) try {
    if (!c || !pod_offset || (n && (!node_names || !out_placed))) return fail(KS_ERR_INVALID, "NULL argument");
    if (pod_offset[0] != 0) return fail(KS_ERR_INVALID, "pod_offset[0] must be 0");
    for (uint64_t d = 0; d < n; d++)
        if (pod_offset[d + 1] < pod_offset[d]) return fail(KS_ERR_INVALID, "pod offsets decrease");
    const uint64_t P = pod_offset[n];
    if (P && (!pods || !out_node_idx)) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    std::vector<int32_t> node(n);
    for (uint64_t d = 0; d < n; d++) { // mis-grouped input is refused before anything is packed
        const char* name = node_names[d];
        if (!name) return fail(KS_ERR_INVALID, "candidate " + std::to_string(d) + ": node name is NULL");
        node[d] = node_index_of(c, name);
        if (node[d] < 0) return fail(KS_ERR_INVALID, "candidate " + std::to_string(d) + ": node \"" + name + "\" is not in the store");
        for (uint64_t i = pod_offset[d]; i < pod_offset[d + 1]; i++)
            if (!ksh_is_pod_bound(&pods[i]) || std::strcmp(pods[i].node_name, name) != 0)
                return fail(KS_ERR_INVALID, "pod " + std::to_string(i) + " (" + nz(pods[i].ns) + "/" + nz(pods[i].name) +
                                                ") has spec.nodeName \"" + (ksh_is_pod_bound(&pods[i]) ? pods[i].node_name : "") +
                                                "\", not its candidate's node \"" + name + "\"");
    }
    int rc = device_ready(c, ks_drain_check, "ks_drain_check");
    if (rc) return rc;
    ks_pods kp;
    rc = pack_batch(c, pods, P, &kp);
    if (rc) return rc;
    ks_drain_candidates kc{n, node.data(), pod_offset};
    return ks_drain_check(c->snap, &kp, &kc, policy, flags, out_placed, out_node_idx, nullptr);
}
KSH_CATCH

int ksh_place_replicas(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const uint32_t* replicas, int policy,
                       ks_replica_plan* out, int32_t* out_node, int64_t* out_score) try {
    if (!c || (n && (!pods || !replicas || !out))) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    int rc = device_ready(c, ks_place_replicas, "ks_place_replicas");
    if (rc) return rc;
    if (n == 0) return KS_OK;
    ks_pods kp;
    rc = pack_batch(c, pods, n, &kp);
    if (rc) return rc;
    return ks_place_replicas(c->snap, &kp, replicas, policy, out, out_node, out_score);
}
KSH_CATCH

// Dense domain ids of one topology key in order of first appearance over the node indices; -1 for a node without it.
// values[d] = the pair id of domain d.
static uint32_t topology_domains(const ksh_context* c, const char* key, int32_t* dom, std::vector<uint32_t>* values) {
    std::unordered_map<uint32_t, int32_t> of_pair; // pair id -> domain
    for (uint32_t n = 0; n < c->N; n++) {
        dom[n] = -1;
        for (uint32_t pid : c->node_pids[n]) {
            if (std::strcmp(c->pairs.str(pid), key) != 0) continue; // "key\0value": the key part ends at the NUL
            auto it = of_pair.emplace(pid, (int32_t)of_pair.size()).first;
            if (it->second == (int32_t)values->size()) values->push_back(pid);
            dom[n] = it->second;
            break; // a node carries a key once
        }
    }
    return (uint32_t)values->size();
}

int ksh_context_topology_domains(const ksh_context* c, const char* key, int32_t* out_node_domain, uint32_t* out_n_domains,
                                 char* names, size_t cap, int64_t* out_name_off) try {
    if (!c || !key || !out_n_domains || (c->N && !out_node_domain)) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    std::vector<uint32_t> values;
    const uint32_t D = topology_domains(c, key, out_node_domain, &values);
    *out_n_domains = D;
    if (!names || !out_name_off) return KS_OK;
    StringList list{names, cap};
    for (uint32_t d = 0; d < D; d++) {
        const char* k = c->pairs.str(values[d]);
        const char* v = k + std::strlen(k) + 1;
        out_name_off[d] = list.append(v, std::strlen(v) + 1);
    }
    return KS_OK;
}
KSH_CATCH

// ksh_place_replicas_spread (multi = false, K = 1) and ksh_place_replicas_spread_multi: existing_offset[t * K + k]
// indexes spec t's existing pods under key k.  A name counts when it is in the store and its node carries every key.
static int place_spread_objects(ksh_context* c, bool multi, const ks_pod_obj* pods, uint64_t n, const uint32_t* replicas,
                                const char* const* keys, uint32_t K, const uint32_t* max_skew, const uint32_t* min_domains,
                                const char* const* existing_node_names, const uint64_t* existing_offset, int policy,
                                ks_spread_plan* out, int32_t* out_node, int64_t* out_score, uint32_t* out_domain_count) {
    if (!c || !keys || (n && (!pods || !replicas || !max_skew || !out))) return fail(KS_ERR_INVALID, "NULL argument");
    if (K == 0 || K > KS_SPREAD_MAX_KEYS)
        return fail(KS_ERR_RANGE, std::to_string(K) + " topology keys (1 to " + std::to_string(KS_SPREAD_MAX_KEYS) + ")");
    for (uint32_t k = 0; k < K; k++)
        if (!keys[k]) return fail(KS_ERR_INVALID, "NULL argument");
    const uint64_t nk = n * K;
    if (existing_offset && existing_offset[nk] && !existing_node_names) return fail(KS_ERR_INVALID, "NULL existing_node_names");
    if (existing_offset)
        for (uint64_t i = 0; i < nk; i++)
            if (existing_offset[i + 1] < existing_offset[i]) return fail(KS_ERR_INVALID, "existing offsets decrease");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    int rc = multi ? device_ready(c, ks_place_replicas_spread_multi, "ks_place_replicas_spread_multi")
                   : device_ready(c, ks_place_replicas_spread, "ks_place_replicas_spread");
    if (rc) return rc;
    if (n == 0) return KS_OK;
    ks_pods kp;
    rc = pack_batch(c, pods, n, &kp);
    if (rc) return rc;
    std::vector<std::vector<int32_t>> dom(K, std::vector<int32_t>(c->N));
    uint32_t Dc[KS_SPREAD_MAX_KEYS] = {}, P[KS_SPREAD_MAX_KEYS] = {};
    uint64_t S = 0;
    bool keyless = false;
    for (uint32_t k = 0; k < K; k++) {
        std::vector<uint32_t> values;
        const uint32_t D = topology_domains(c, keys[k], dom[k].data(), &values);
        keyless |= D == 0;
        // no node carries the key: no domain is eligible, and a single empty domain gives exactly that
        Dc[k] = std::max(D, 1u);
        P[k] = (uint32_t)S;
        S += Dc[k];
    }
    std::vector<uint32_t> existing;
    if (existing_offset) {
        if (n * S > KS_SPREAD_MAX_COUNTS) return fail(KS_ERR_RANGE, "too many specs x domains of existing counts (at most 2^26)");
        existing.assign(n * S, 0);
        for (uint64_t t = 0; t < n; t++)
            for (uint32_t k = 0; k < K; k++)
                for (uint64_t i = existing_offset[t * K + k]; i < existing_offset[t * K + k + 1]; i++) {
                    const int32_t idx = existing_node_names[i] ? node_index_of(c, existing_node_names[i]) : -1;
                    if (idx < 0) continue; // unknown: not counted
                    bool all = true;
                    for (uint32_t k2 = 0; k2 < K; k2++) all &= dom[k2][idx] >= 0;
                    if (all) existing[t * S + P[k] + (uint32_t)dom[k][idx]]++; // keyless: not counted
                }
    }
    uint32_t* counts = keyless ? nullptr : out_domain_count;
    if (!multi) {
        ks_spread sp{Dc[0], dom[0].data(), max_skew, min_domains, existing_offset ? existing.data() : nullptr};
        return ks_place_replicas_spread(c->snap, &kp, replicas, &sp, policy, out, out_node, out_score, counts);
    }
    ks_spread_multi sp{};
    sp.n_keys = K;
    for (uint32_t k = 0; k < K; k++) {
        sp.n_domains[k] = Dc[k];
        sp.node_domain[k] = dom[k].data();
    }
    sp.max_skew = max_skew;
    sp.min_domains = min_domains;
    sp.existing = existing_offset ? existing.data() : nullptr;
    return ks_place_replicas_spread_multi(c->snap, &kp, replicas, &sp, policy, out, out_node, out_score, counts);
}

int ksh_place_replicas_spread(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const uint32_t* replicas,
                              const char* topology_key, const uint32_t* max_skew, const uint32_t* min_domains,
                              const char* const* existing_node_names, const uint64_t* existing_offset, int policy,
                              ks_spread_plan* out, int32_t* out_node, int64_t* out_score, uint32_t* out_domain_count) try {
    return place_spread_objects(c, false, pods, n, replicas, topology_key ? &topology_key : nullptr, 1, max_skew,
                                min_domains, existing_node_names, existing_offset, policy, out, out_node, out_score,
                                out_domain_count);
}
KSH_CATCH

int ksh_place_replicas_spread_multi(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const uint32_t* replicas,
                                    const char* const* topology_keys, uint32_t n_keys, const uint32_t* max_skew,
                                    const uint32_t* min_domains, const char* const* existing_node_names,
                                    const uint64_t* existing_offset, int policy, ks_spread_plan* out, int32_t* out_node,
                                    int64_t* out_score, uint32_t* out_domain_count) try {
    return place_spread_objects(c, true, pods, n, replicas, topology_keys, n_keys, max_skew, min_domains,
                                existing_node_names, existing_offset, policy, out, out_node, out_score, out_domain_count);
}
KSH_CATCH

// ---- taints and node affinity (ks_node_bind, DESIGN.md 5p) ----
// The packed rules of one call over the node store, and the arrays its pointers reach
struct CompiledNodeRules {
    ks_node_rules r{};
    std::vector<uint64_t> hard, soft, tol_h, tol_s, set_off, sets;
    std::vector<std::vector<int32_t>> dom;
    std::vector<uint32_t> expr_key, term_w, term_off;
    std::vector<int32_t> owner;
};

// Go's strconv.ParseInt(s, 10, 64)
static bool parse_int64(const char* s, int64_t* v) {
    if (!s || !*s) return false;
    size_t i = 0;
    const bool neg = s[0] == '-';
    if (s[0] == '+' || s[0] == '-') i = 1;
    if (!s[i]) return false;
    u128 m = 0;
    for (; s[i]; i++) {
        if (s[i] < '0' || s[i] > '9') return false;
        m = m * 10 + (unsigned)(s[i] - '0');
        if (m > ((u128)1 << 63)) return false;
    }
    if (!neg && m > (u128)INT64_MAX) return false;
    *v = neg ? (int64_t)(0 - (uint64_t)m) : (int64_t)m;
    return true;
}

static bool tolerates(const ksh_toleration& t, const std::array<std::string, 3>& taint) {
    const std::string op = nz(t.op), eff = nz(t.effect), key = nz(t.key);
    if (!eff.empty() && eff != taint[2]) return false;
    if (!key.empty() && key != taint[0]) return false;
    if (op == "Exists") return true;
    return nz(t.value) == taint[1]; // "" or Equal
}

// The node side of a rule compilation: the store's nodes (store_nodes) or a call's node templates.  taints_of(n) is node
// n's spec.taints (NULL: none); domains(key, dom, values) numbers the key's values over the nodes as topology_domains
// does, dom[n] = -1 for a node without the key, values[d] = domain d's value.
using Taint = std::array<std::string, 3>; // key, value, effect
struct RuleNodes {
    uint32_t N = 0;
    const char* what = ""; // in the too-many-taints message
    std::function<const std::vector<Taint>*(uint32_t)> taints_of;
    std::function<void(const std::string&, int32_t*, std::vector<std::string>*)> domains;
};

static RuleNodes store_nodes(const ksh_context* c) {
    RuleNodes nodes;
    nodes.N = c->N;
    nodes.what = "the store's nodes";
    nodes.taints_of = [c](uint32_t n) -> const std::vector<Taint>* {
        const auto it = c->taints.find(c->names.str(c->idx2nameid[n]));
        return it == c->taints.end() ? nullptr : &it->second;
    };
    nodes.domains = [c](const std::string& key, int32_t* dom, std::vector<std::string>* values) {
        std::vector<uint32_t> pids;
        topology_domains(c, key.c_str(), dom, &pids);
        for (const uint32_t pid : pids) {
            const char* k = c->pairs.str(pid);
            values->emplace_back(k + std::strlen(k) + 1);
        }
    };
    return nodes;
}

static int compile_rules_over(const RuleNodes& nodes, uint32_t G, const ksh_node_rules* in, CompiledNodeRules* out) {
    const ksh_node_rules none{};
    if (!in) in = &none;
    const uint32_t N = nodes.N, T = in->n_terms;
    if (in->toleration_offset && in->toleration_offset[G] && !in->tolerations) return fail(KS_ERR_INVALID, "NULL tolerations");
    if (T && (!in->term_owner || !in->term_weight || !in->term_req_offset))
        return fail(KS_ERR_INVALID, "NULL term_owner, term_weight or term_req_offset");
    if (T && in->term_req_offset[T] && !in->requirements) return fail(KS_ERR_INVALID, "NULL requirements");
    if (in->toleration_offset)
        for (uint32_t g = 0; g < G; g++) {
            if (in->toleration_offset[g + 1] < in->toleration_offset[g])
                return fail(KS_ERR_INVALID, "toleration offsets decrease");
            for (uint64_t i = in->toleration_offset[g]; i < in->toleration_offset[g + 1]; i++) {
                const std::string op = nz(in->tolerations[i].op);
                if (op != "" && op != "Equal" && op != "Exists")
                    return fail(KS_ERR_INVALID, "group " + std::to_string(g) + ": toleration operator \"" + op + "\"");
                if (op == "Exists" && *nz(in->tolerations[i].value))
                    return fail(KS_ERR_INVALID, "group " + std::to_string(g) + ": Exists toleration with a value");
            }
        }
    std::vector<std::string> keys; // requirement keys in order of first appearance
    for (uint32_t t = 0; t < T; t++) {
        if (in->term_owner[t] < 0 || in->term_owner[t] >= (int64_t)G)
            return fail(KS_ERR_INVALID, "node-affinity term " + std::to_string(t) + ": owner outside [0, n_groups)");
        if (in->term_weight[t] > 100) return fail(KS_ERR_INVALID, "node-affinity term " + std::to_string(t) + ": weight above 100");
        if (in->term_req_offset[t + 1] < in->term_req_offset[t]) return fail(KS_ERR_INVALID, "requirement offsets decrease");
        for (uint64_t i = in->term_req_offset[t]; i < in->term_req_offset[t + 1]; i++) {
            const ksh_node_selector_requirement& q = in->requirements[i];
            const std::string op = nz(q.op), where = "requirement " + std::to_string(i) + " (" + op + "): ";
            if (!q.key || !*q.key) return fail(KS_ERR_INVALID, where + "empty key");
            if (q.n_values && !q.values) return fail(KS_ERR_INVALID, where + "NULL values");
            for (uint32_t v = 0; v < q.n_values; v++)
                if (!q.values[v]) return fail(KS_ERR_INVALID, where + "NULL value");
            int64_t x;
            if (op == "In" || op == "NotIn") {
                if (!q.n_values) return fail(KS_ERR_INVALID, where + "no values");
            } else if (op == "Exists" || op == "DoesNotExist") {
                if (q.n_values) return fail(KS_ERR_INVALID, where + "values given");
            } else if (op == "Gt" || op == "Lt") {
                if (q.n_values != 1 || !parse_int64(q.values[0], &x))
                    return fail(KS_ERR_INVALID, where + "needs exactly one integer value");
            } else {
                return fail(KS_ERR_INVALID, where + "unknown operator");
            }
            if (std::find(keys.begin(), keys.end(), q.key) == keys.end()) keys.emplace_back(q.key);
        }
    }
    if (keys.size() > KS_NODE_RULES_MAX_KEYS)
        return fail(KS_ERR_RANGE, std::to_string(keys.size()) + " node-affinity keys (at most " +
                                      std::to_string(KS_NODE_RULES_MAX_KEYS) + ")");
    // taints: the distinct (key, value, effect) triples of the nodes, numbered in node order
    std::vector<Taint> triples;
    out->hard.assign(N, 0);
    out->soft.assign(N, 0);
    for (uint32_t n = 0; n < N; n++) {
        const std::vector<Taint>* ts = nodes.taints_of(n);
        if (!ts) continue;
        for (const auto& t : *ts) {
            size_t b = std::find(triples.begin(), triples.end(), t) - triples.begin();
            if (b == triples.size()) {
                if (b == KS_NODE_RULES_MAX_TAINTS)
                    return fail(KS_ERR_RANGE, std::string("more than 64 distinct taints on ") + nodes.what);
                triples.push_back(t);
            }
            (t[2] == "PreferNoSchedule" ? out->soft : out->hard)[n] |= 1ull << b;
        }
    }
    out->tol_h.assign(G, 0);
    out->tol_s.assign(G, 0);
    for (uint32_t g = 0; g < G && in->toleration_offset; g++)
        for (size_t b = 0; b < triples.size(); b++)
            for (uint64_t i = in->toleration_offset[g]; i < in->toleration_offset[g + 1]; i++) {
                const ksh_toleration& t = in->tolerations[i];
                if (!tolerates(t, triples[b])) continue;
                if (triples[b][2] != "PreferNoSchedule") out->tol_h[g] |= 1ull << b;
                else if (!*nz(t.effect) || std::string(t.effect) == "PreferNoSchedule") out->tol_s[g] |= 1ull << b;
            }
    // node affinity: each key's domains over the nodes, each requirement a set over them plus the "absent" bit
    std::vector<std::vector<std::string>> values(keys.size());
    out->dom.assign(keys.size(), std::vector<int32_t>(N));
    for (size_t k = 0; k < keys.size(); k++) nodes.domains(keys[k], out->dom[k].data(), &values[k]);
    out->set_off.push_back(0);
    out->term_off.push_back(0);
    for (uint32_t t = 0; t < T; t++) {
        for (uint64_t i = in->term_req_offset[t]; i < in->term_req_offset[t + 1]; i++) {
            const ksh_node_selector_requirement& q = in->requirements[i];
            const uint32_t k = (uint32_t)(std::find(keys.begin(), keys.end(), q.key) - keys.begin());
            const uint64_t D = values[k].size(), base = out->sets.size();
            out->sets.resize(base + (D + 64) / 64, 0);
            const std::string op = q.op;
            int64_t lim = 0;
            if (op == "Gt" || op == "Lt") parse_int64(q.values[0], &lim);
            for (uint64_t d = 0; d <= D; d++) {
                bool in_set;
                if (d == D) { // the node lacks the key
                    in_set = op == "NotIn" || op == "DoesNotExist";
                } else {
                    const std::string& v = values[k][d];
                    bool listed = false;
                    for (uint32_t j = 0; j < q.n_values; j++) listed |= v == q.values[j];
                    int64_t x;
                    in_set = op == "In"       ? listed
                             : op == "NotIn"  ? !listed
                             : op == "Exists" ? true
                             : op == "Gt"     ? parse_int64(v.c_str(), &x) && x > lim
                             : op == "Lt"     ? parse_int64(v.c_str(), &x) && x < lim
                                              : false;
                }
                if (in_set) out->sets[base + d / 64] |= 1ull << (d % 64);
            }
            out->set_off.push_back(out->sets.size());
            out->expr_key.push_back(k);
        }
        out->term_off.push_back((uint32_t)out->expr_key.size());
        out->owner.push_back(in->term_owner[t]);
        out->term_w.push_back(in->term_weight[t]);
    }
    ks_node_rules& r = out->r;
    r.n_taints = (uint32_t)triples.size();
    r.node_taint_hard = out->hard.data();
    r.node_taint_soft = out->soft.data();
    r.tolerate_hard = out->tol_h.data();
    r.tolerate_soft = out->tol_s.data();
    r.n_keys = (uint32_t)keys.size();
    for (size_t k = 0; k < keys.size(); k++) {
        r.n_domains[k] = (uint32_t)values[k].size();
        r.node_domain[k] = out->dom[k].data();
    }
    r.n_exprs = (uint32_t)out->expr_key.size();
    r.expr_key = out->expr_key.data();
    r.expr_set_offset = out->set_off.data();
    r.expr_set = out->sets.data();
    r.n_terms = T;
    r.term_owner = out->owner.data();
    r.term_weight = out->term_w.data();
    r.term_expr_offset = out->term_off.data();
    r.weight_taint = in == &none ? 3 : in->weight_taint;
    r.weight_node_affinity = in == &none ? 2 : in->weight_node_affinity;
    return KS_OK;
}

// over the store's nodes and their recorded taints
static int compile_node_rules(ksh_context* c, uint32_t G, const ksh_node_rules* in, CompiledNodeRules* out) {
    return compile_rules_over(store_nodes(c), G, in, out);
}

// ---- extended resources (ks_fit_bind, DESIGN.md 5r) ----
// The scalar resources of a pending batch: "pods", then every other name some pod of the batch requests with a non-zero
// quantity, in order of first request; node_free [R * N] = allocatable (0 when the node does not list the name) minus
// the requests of the rows bound on the node (for "pods", the rows themselves); pod_req [P * R] (1 for "pods").
struct CompiledResources {
    std::vector<uint32_t> ids; // resource ids, ids[0] = "pods"
    std::vector<int64_t> node_free, pod_req;
};

static std::string pod_key(const ks_pod_obj* pod) { return std::string(nz(pod->ns)) + "/" + nz(pod->name); }

// The error of a recorded quantity e of `who` ("pod 'ns/name'", "node 'name'", ...): KS_ERR_PARSE for a quantity that
// does not parse, KS_ERR_RANGE for a pod's requests that sum past int64
static int ext_error(const ksh_context* c, const std::string& who, const char* what, const ExtQty& e) {
    if (e.err == EXT_OVERFLOW)
        return fail(KS_ERR_RANGE, who + ": its " + c->res_name[e.res] + " requests sum past int64");
    return fail(KS_ERR_PARSE, who + ": cannot convert its " + what + c->res_name[e.res] + " to an integer");
}

// The batch side of compile_resources: ids, and pod_req [n * R]
static int batch_resources(ksh_context* c, const ks_pod_obj* pods, uint64_t n, CompiledResources* out) {
    const uint32_t pods_id = res_id(c, "pods");
    out->ids.assign(1, pods_id);
    std::vector<std::vector<ExtQty>> req(n);
    for (uint64_t p = 0; p < n; p++) {
        req[p] = pod_ext(c, &pods[p]);
        for (const ExtQty& e : req[p]) {
            if (e.res == pods_id) continue; // the pod count is not requested: every pod counts 1
            if (e.err) return ext_error(c, "pod '" + pod_key(&pods[p]) + "'", "request of ", e);
            if (e.v < 0)
                return fail(KS_ERR_RANGE, "pod '" + pod_key(&pods[p]) + "': negative " + c->res_name[e.res] + " request");
            if (std::find(out->ids.begin(), out->ids.end(), e.res) == out->ids.end()) out->ids.push_back(e.res);
        }
    }
    const size_t R = out->ids.size();
    if (R > KS_BIND_MAX_RESOURCES)
        return fail(KS_ERR_RANGE, std::to_string(R) + " resources in one batch, \"pods\" included (at most " +
                                      std::to_string(KS_BIND_MAX_RESOURCES) + "): split the batch");
    std::vector<int32_t> col(c->res_name.size(), -1);
    for (size_t r = 0; r < R; r++) col[out->ids[r]] = (int32_t)r;
    out->pod_req.assign(n * R, 0);
    for (uint64_t p = 0; p < n; p++) {
        out->pod_req[p * R] = 1;
        for (const ExtQty& e : req[p])
            if (col[e.res] > 0) out->pod_req[p * R + (size_t)col[e.res]] = e.v;
    }
    return KS_OK;
}

static int compile_resources(ksh_context* c, const ks_pod_obj* pods, uint64_t n, CompiledResources* out) {
    const int rc = batch_resources(c, pods, n, out);
    if (rc) return rc;
    const size_t R = out->ids.size(), N = c->N;
    std::vector<int32_t> col(c->res_name.size(), -1);
    for (size_t r = 0; r < R; r++) col[out->ids[r]] = (int32_t)r;
    out->node_free.assign(R * N, 0);
    for (size_t i = 0; i < N; i++)
        for (const ExtQty& e : c->node_ext[i]) {
            if (col[e.res] < 0) continue;
            if (e.err)
                return ext_error(c, std::string("node '") + c->names.str(c->idx2nameid[i]) + "'", "allocatable ", e);
            out->node_free[(size_t)col[e.res] * N + i] = e.v;
        }
    for (size_t b = 0; b < c->bnode.size(); b++) {
        const size_t node = (size_t)c->bnode[b];
        int64_t& pc = out->node_free[node];
        bool over = __builtin_sub_overflow(pc, 1, &pc);
        for (const ExtQty& e : c->bext[b]) {
            if (e.res >= col.size() || col[e.res] <= 0) continue;
            if (e.err)
                return ext_error(c, "bound pod '" + std::string(c->bkeys.data() + c->boff[b], c->blen[b]) + "'",
                                 "request of ", e);
            int64_t& f = out->node_free[(size_t)col[e.res] * N + node];
            over |= __builtin_sub_overflow(f, e.v, &f);
        }
        if (over) return fail(KS_ERR_RANGE, "free resources of a node overflow int64");
    }
    return KS_OK;
}

// The bind call behind each reconcile mode (ks_spread_bind to ks_gang_fit_bind), and its refusal words per pod: the
// word of each reason, -1 where the mode has none.  Node affinity follows taint.
enum ReconcileMode { RM_SPREAD, RM_AFFINITY, RM_PROFILE, RM_NODES, RM_FIT, RM_FIT_GANGS };
struct RefusalWords { size_t n; int res, taint, spread, aff; };
static const RefusalWords REFUSAL_WORDS[] = {{1, -1, -1, 0, -1}, {2, -1, -1, 0, 1}, {2, -1, -1, 0, 1},
                                             {4, -1, 0, 2, 3},   {5, 0, 1, 3, 4},    {5, 0, 1, 3, 4}};

// What a reconcile mode adds to reconcile_spread's arguments: the soft terms (PROFILE on), the node rules (NODES on) and
// the gangs (FIT_GANGS)
struct ReconcileRequest {
    ReconcileMode mode = RM_SPREAD;
    const ks_bind_scoring* sc = nullptr;
    const ksh_node_rules* nr = nullptr;
    const uint64_t* gang_offset = nullptr;
    uint64_t n_gangs = 0;
    const uint32_t* min_member = nullptr;
    uint32_t* out_placed = nullptr;
};

// The mode's device entry: with kp NULL, device_ready for it; else the call over the packed batch, which commits
// capacity on the device
static int bind_device(ksh_context* c, ReconcileMode m, const ks_pods* kp, const int32_t* group, uint32_t G,
                       const ks_spread_multi* sp, const ks_pod_affinity* pa, const ks_bind_scoring* sc,
                       const ks_node_rules* nr, const ks_bind_resources* br, const ks_gangs* kg, int policy,
                       int32_t* idx, uint32_t* refused, uint32_t* placed) {
    switch (m) {
    case RM_SPREAD:
        if (!kp) return device_ready(c, ks_spread_bind, "ks_spread_bind");
        return ks_spread_bind(c->snap, kp, group, G, sp, policy, idx, nullptr, refused, nullptr);
    case RM_AFFINITY:
        if (!kp) return device_ready(c, ks_affinity_bind, "ks_affinity_bind");
        return ks_affinity_bind(c->snap, kp, group, G, sp, pa, policy, idx, nullptr, refused, nullptr);
    case RM_PROFILE:
        if (!kp) return device_ready(c, ks_profile_bind, "ks_profile_bind");
        return ks_profile_bind(c->snap, kp, group, G, sp, pa, sc, policy, idx, nullptr, nullptr, refused, nullptr,
                               nullptr);
    case RM_NODES:
        if (!kp) return device_ready(c, ks_node_bind, "ks_node_bind");
        return ks_node_bind(c->snap, kp, group, G, sp, pa, sc, nr, policy, idx, nullptr, nullptr, refused, nullptr,
                            nullptr);
    case RM_FIT:
        if (!kp) return device_ready(c, ks_fit_bind, "ks_fit_bind");
        return ks_fit_bind(c->snap, kp, group, G, sp, pa, sc, nr, br, policy, idx, nullptr, nullptr, refused, nullptr,
                           nullptr, nullptr);
    case RM_FIT_GANGS:
        if (!kp) return device_ready(c, ks_gang_fit_bind, "ks_gang_fit_bind");
        return ks_gang_fit_bind(c->snap, kp, group, G, sp, pa, sc, nr, br, kg, policy, idx, nullptr, nullptr, refused,
                                nullptr, nullptr, nullptr, placed);
    }
    return fail(KS_ERR_INVALID, "bad reconcile mode");
}

// The gangs' part of a batch (ksh_reconcile_fit_gangs): keeps of todo, sub and sub_group the pods of the gangs that can
// still commit, as sub-gang k = [sub_off[k], sub_off[k + 1]) of gang sub_gang[k] needing sub_min[k] more pods.  Running
// members count toward min_member, as in ksh_reconcile_gangs; a gang with too few schedulable members is not tried.
static void cut_gangs(const ReconcileRequest& m, int32_t* out_status, std::vector<uint64_t>& todo,
                      std::vector<ks_pod_obj>& sub, std::vector<int32_t>& sub_group, std::vector<uint64_t>& sub_off,
                      std::vector<uint64_t>& sub_gang, std::vector<uint32_t>& sub_min) {
    std::vector<uint64_t> keep;
    std::vector<ks_pod_obj> keep_pods;
    std::vector<int32_t> keep_group;
    for (uint64_t j = 0, t = 0; j < m.n_gangs; j++) {
        uint32_t bound = 0; // running members of the gang
        for (uint64_t i = m.gang_offset[j]; i < m.gang_offset[j + 1]; i++) bound += out_status[i] == KSH_RECONCILE_OK;
        const size_t first = t;
        while (t < todo.size() && todo[t] < m.gang_offset[j + 1]) t++;
        const uint32_t need = m.min_member[j] > bound ? m.min_member[j] - bound : 0;
        if (t == first) continue;
        if (need > t - first) { // too few schedulable members: the gang cannot commit, nothing is tried
            for (size_t k = first; k < t; k++) out_status[todo[k]] = KSH_RECONCILE_GANG_UNSATISFIED;
            continue;
        }
        for (size_t k = first; k < t; k++) {
            keep.push_back(todo[k]);
            keep_pods.push_back(sub[k]);
            keep_group.push_back(sub_group[k]);
        }
        sub_off.push_back(keep.size());
        sub_gang.push_back(j);
        sub_min.push_back(need);
    }
    todo.swap(keep);
    sub.swap(keep_pods);
    sub_group.swap(keep_group);
}

// reconcile() under topology spread: ksh_reconcile_batch's filtering, then the mode's bind call over the pods that go to
// the device, each in its group.  Group g's existing pods under key k count when their node is in the store and carries
// key k and every key g constrains.  AFFINITY on: the terms and the existing pods whose node is in the store; max_skew may
// then be NULL.  PROFILE on: the soft terms of m.sc, whose counts start from the same existing counts.  NODES on: the
// node rules.  FIT on: the batch's resources.  FIT_GANGS: one sub-gang per gang, as cut_gangs leaves them.
static int reconcile_spread(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const int32_t* group, uint32_t n_groups,
                            const char* const* topology_keys, uint32_t K, const uint32_t* max_skew,
                            const uint32_t* min_domains, const char* const* existing_node_names,
                            const uint64_t* existing_offset, const ksh_pod_affinity* aff, int policy, int32_t* out_status,
                            int32_t* out_node_idx, char* json, size_t cap, int64_t* out_json_off,
                            const ReconcileRequest& m) {
    if (!c || !topology_keys || (n && (!pods || !group || !out_status || !out_node_idx)) || (n_groups && !max_skew && !aff))
        return fail(KS_ERR_INVALID, "NULL argument");
    if (m.gang_offset) { // as ksh_reconcile_gangs checks them, without its size limit
        if (m.n_gangs && !m.min_member) return fail(KS_ERR_INVALID, "NULL argument");
        const int rc = check_cut("gang", m.gang_offset, m.n_gangs, m.min_member, n, UINT64_MAX);
        if (rc) return rc;
    }
    if (K == 0 || K > KS_SPREAD_MAX_KEYS)
        return fail(KS_ERR_RANGE, std::to_string(K) + " topology keys (1 to " + std::to_string(KS_SPREAD_MAX_KEYS) + ")");
    for (uint32_t k = 0; k < K; k++)
        if (!topology_keys[k]) return fail(KS_ERR_INVALID, "NULL argument");
    for (uint64_t i = 0; i < n; i++)
        if (group[i] < -1 || group[i] >= (int64_t)n_groups)
            return fail(KS_ERR_INVALID, "pod " + std::to_string(i) + ": group outside [-1, n_groups)");
    const uint64_t gk = (uint64_t)n_groups * K;
    if (existing_offset && existing_offset[gk] && !existing_node_names) return fail(KS_ERR_INVALID, "NULL existing_node_names");
    if (existing_offset)
        for (uint64_t i = 0; i < gk; i++)
            if (existing_offset[i + 1] < existing_offset[i]) return fail(KS_ERR_INVALID, "existing offsets decrease");
    if (aff && aff->n_existing && (!aff->existing_group || !aff->existing_node_name))
        return fail(KS_ERR_INVALID, "NULL existing_group or existing_node_name");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    int rc = bind_device(c, m.mode, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr,
                         nullptr, nullptr);
    if (rc) return rc;
    std::vector<uint64_t> todo;
    std::vector<ks_pod_obj> sub; // the pods that go to the device, in arrival order, and their groups
    std::vector<int32_t> sub_group;
    for (uint64_t i = 0; i < n; i++) {
        out_node_idx[i] = -1;
        if (out_json_off) out_json_off[i] = -1;
        out_status[i] = reconcile_status(c, &pods[i]);
        if (out_status[i] != KSH_RECONCILE_NO_NODE_FOUND) continue;
        todo.push_back(i);
        sub.push_back(pods[i]);
        sub_group.push_back(group[i]);
    }
    std::vector<uint64_t> sub_off{0}, sub_gang; // FIT_GANGS: the sub-gangs
    std::vector<uint32_t> sub_min;
    if (m.out_placed)
        for (uint64_t j = 0; j < m.n_gangs; j++) m.out_placed[j] = 0;
    if (m.gang_offset) cut_gangs(m, out_status, todo, sub, sub_group, sub_off, sub_gang, sub_min);
    CompiledNodeRules cr;
    if (m.mode >= RM_NODES) { // compiled before anything is bound, so a bad rule fails the whole call
        rc = compile_node_rules(c, n_groups, m.nr, &cr);
        if (rc) return rc;
    }
    if (todo.empty()) return KS_OK;
    CompiledResources res;
    if (m.mode >= RM_FIT) { // before the device, so a bad quantity fails the whole call
        rc = compile_resources(c, sub.data(), sub.size(), &res);
        if (rc) return rc;
    }
    ks_pods kp;
    rc = pack_batch(c, sub.data(), sub.size(), &kp);
    if (rc) return rc;
    std::vector<std::vector<int32_t>> dom(K, std::vector<int32_t>(c->N));
    ks_spread_multi sp{};
    uint32_t P[KS_SPREAD_MAX_KEYS] = {};
    uint64_t S = 0;
    for (uint32_t k = 0; k < K; k++) {
        std::vector<uint32_t> values;
        // no node carries the key: a single empty domain, so no node is eligible under it
        sp.n_domains[k] = std::max(topology_domains(c, topology_keys[k], dom[k].data(), &values), 1u);
        sp.node_domain[k] = dom[k].data();
        P[k] = (uint32_t)S;
        S += sp.n_domains[k];
    }
    std::vector<uint32_t> existing;
    if (existing_offset) {
        if (n_groups * S > KS_SPREAD_MAX_COUNTS) return fail(KS_ERR_RANGE, "too many groups x domains of counts (at most 2^26)");
        existing.assign(n_groups * S, 0);
        for (uint64_t g = 0; g < n_groups; g++)
            for (uint32_t k = 0; k < K; k++)
                for (uint64_t i = existing_offset[g * K + k]; i < existing_offset[g * K + k + 1]; i++) {
                    const int32_t idx = existing_node_names[i] ? node_index_of(c, existing_node_names[i]) : -1;
                    if (idx < 0) continue; // unknown: not counted
                    bool all = dom[k][idx] >= 0;
                    for (uint32_t k2 = 0; k2 < K; k2++) all &= !max_skew || max_skew[g * K + k2] == 0 || dom[k2][idx] >= 0;
                    if (all) existing[g * S + P[k] + (uint32_t)dom[k][idx]]++;
                }
    }
    sp.n_keys = K;
    sp.max_skew = max_skew;
    sp.min_domains = min_domains;
    sp.existing = existing_offset ? existing.data() : nullptr;
    ks_pod_affinity pa{};
    std::vector<int32_t> eg, en; // the existing pods whose node is in the store
    if (aff) {
        pa = {aff->n_terms, aff->owner, aff->kind, aff->key, aff->target_offset, aff->target, 0, nullptr, nullptr};
        for (uint64_t e = 0; e < aff->n_existing; e++) {
            const int32_t at = aff->existing_node_name[e] ? node_index_of(c, aff->existing_node_name[e]) : -1;
            if (at < 0) continue;
            eg.push_back(aff->existing_group[e]);
            en.push_back(at);
        }
        pa.n_existing = eg.size();
        pa.existing_group = eg.data();
        pa.existing_node = en.data();
    }
    const RefusalWords& L = REFUSAL_WORDS[m.mode];
    std::vector<int32_t> idx(sub.size(), -1);
    std::vector<uint32_t> refused(sub.size() * L.n, 0);
    std::vector<uint32_t> placed(sub_gang.size());
    const ks_bind_resources br{(uint32_t)res.ids.size(), res.node_free.data(), res.pod_req.data()};
    const ks_gangs kg{sub_gang.size(), sub_off.data(), sub_min.data()};
    rc = bind_device(c, m.mode, &kp, sub_group.data(), n_groups, &sp, &pa, m.sc, &cr.r, &br, &kg, policy, idx.data(),
                     refused.data(), placed.data());
    if (rc) {
        c->dirty = true; // the host list is the truth
        return rc;
    }
    StringList bodies{json, cap};
    std::vector<uint8_t> rolled(todo.size(), 0); // the pods of the sub-gangs that rolled back
    for (size_t k = 0; k < sub_gang.size(); k++) {
        if (m.out_placed) m.out_placed[sub_gang[k]] = placed[k];
        if (placed[k] < sub_min[k]) std::fill(rolled.begin() + sub_off[k], rolled.begin() + sub_off[k + 1], 1);
    }
    for (size_t k = 0; k < todo.size(); k++) {
        const uint64_t i = todo[k];
        const uint32_t* w = &refused[k * L.n];
        if (rolled[k])
            out_status[i] = KSH_RECONCILE_GANG_UNSATISFIED;
        else if (idx[k] >= 0)
            commit_bind(c, &pods[i], idx[k], kp.req_cpu[k], kp.req_mem[k], &out_status[i], &out_node_idx[i], bodies,
                        json && out_json_off ? &out_json_off[i] : nullptr);
        else if (L.res >= 0 && w[L.res] > 0 && w[L.taint] + w[L.taint + 1] + w[L.spread] + w[L.aff] == 0)
            out_status[i] = KSH_RECONCILE_INSUFFICIENT_RESOURCES;
        else if (L.taint >= 0 && w[L.taint] + w[L.taint + 1] > 0 && w[L.spread] == 0 && w[L.aff] == 0)
            out_status[i] = KSH_RECONCILE_NODE_RULES_UNSATISFIED;
        else if (w[L.spread] > 0)
            out_status[i] = KSH_RECONCILE_SPREAD_UNSATISFIED;
        else if (L.aff >= 0 && w[L.aff] > 0)
            out_status[i] = KSH_RECONCILE_AFFINITY_UNSATISFIED;
    }
    return KS_OK;
}

int ksh_reconcile_spread(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const int32_t* group, uint32_t n_groups,
                         const char* const* topology_keys, uint32_t K, const uint32_t* max_skew,
                         const uint32_t* min_domains, const char* const* existing_node_names,
                         const uint64_t* existing_offset, int policy, int32_t* out_status, int32_t* out_node_idx,
                         char* json, size_t cap, int64_t* out_json_off) try {
    return reconcile_spread(c, pods, n, group, n_groups, topology_keys, K, max_skew, min_domains, existing_node_names,
                            existing_offset, nullptr, policy, out_status, out_node_idx, json, cap, out_json_off,
                            {RM_SPREAD});
}
KSH_CATCH

int ksh_reconcile_affinity(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const int32_t* group, uint32_t n_groups,
                           const char* const* topology_keys, uint32_t K, const uint32_t* max_skew,
                           const uint32_t* min_domains, const char* const* existing_node_names,
                           const uint64_t* existing_offset, const ksh_pod_affinity* aff, int policy,
                           int32_t* out_status, int32_t* out_node_idx, char* json, size_t cap, int64_t* out_json_off) try {
    const ksh_pod_affinity none{};
    return reconcile_spread(c, pods, n, group, n_groups, topology_keys, K, max_skew, min_domains, existing_node_names,
                            existing_offset, aff ? aff : &none, policy, out_status, out_node_idx, json, cap,
                            out_json_off, {RM_AFFINITY});
}
KSH_CATCH

int ksh_reconcile_profile(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const int32_t* group, uint32_t n_groups,
                          const char* const* topology_keys, uint32_t K, const uint32_t* max_skew,
                          const uint32_t* min_domains, const char* const* existing_node_names,
                          const uint64_t* existing_offset, const ksh_pod_affinity* aff, const ks_bind_scoring* scoring,
                          int policy, int32_t* out_status, int32_t* out_node_idx, char* json, size_t cap,
                          int64_t* out_json_off) try {
    if (!scoring) return fail(KS_ERR_INVALID, "NULL scoring");
    const ksh_pod_affinity none{};
    return reconcile_spread(c, pods, n, group, n_groups, topology_keys, K, max_skew, min_domains, existing_node_names,
                            existing_offset, aff ? aff : &none, policy, out_status, out_node_idx, json, cap,
                            out_json_off, {RM_PROFILE, scoring});
}
KSH_CATCH

int ksh_context_set_node_taints(ksh_context* c, const char* const* node_names, const uint64_t* taint_offset,
                                const ksh_taint* taints, uint64_t n) try {
    if (!c || (n && (!node_names || !taint_offset)) || (n && taint_offset[n] && !taints))
        return fail(KS_ERR_INVALID, "NULL argument");
    for (uint64_t i = 0; i < n; i++) {
        if (!node_names[i]) return fail(KS_ERR_INVALID, "NULL node name");
        if (taint_offset[i + 1] < taint_offset[i]) return fail(KS_ERR_INVALID, "taint offsets decrease");
        for (uint64_t t = taint_offset[i]; t < taint_offset[i + 1]; t++) {
            const std::string e = nz(taints[t].effect);
            if (!taints[t].key || !*taints[t].key || (e != "NoSchedule" && e != "PreferNoSchedule" && e != "NoExecute"))
                return fail(KS_ERR_INVALID, "taint " + std::to_string(t) + ": empty key or effect \"" + e + "\"");
        }
    }
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    for (uint64_t i = 0; i < n; i++) {
        if (node_index_of(c, node_names[i]) < 0) continue; // unknown: ignored
        auto& list = c->taints[node_names[i]];
        list.clear();
        for (uint64_t t = taint_offset[i]; t < taint_offset[i + 1]; t++)
            list.push_back({taints[t].key, nz(taints[t].value), taints[t].effect});
    }
    return KS_OK;
}
KSH_CATCH

int ksh_compile_node_rules(ksh_context* c, uint32_t G, const ksh_node_rules* rules, uint8_t* out_hard,
                           uint8_t* out_affinity, uint32_t* out_soft, uint32_t* out_preferred) try {
    if (!c) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    CompiledNodeRules cr;
    const int rc = compile_node_rules(c, G, rules, &cr);
    if (rc) return rc;
    const ks_node_rules& r = cr.r;
    const uint32_t N = c->N;
    auto match = [&](uint32_t t, uint32_t n) {
        if (r.term_expr_offset[t + 1] == r.term_expr_offset[t]) return false; // no expression: matches nothing
        for (uint32_t x = r.term_expr_offset[t]; x < r.term_expr_offset[t + 1]; x++) {
            const uint32_t k = r.expr_key[x];
            const int32_t d = r.node_domain[k][n];
            const uint64_t b = d < 0 ? r.n_domains[k] : (uint64_t)d;
            if (!(r.expr_set[r.expr_set_offset[x] + b / 64] >> (b % 64) & 1)) return false;
        }
        return true;
    };
    for (uint32_t g = 0; g < G; g++)
        for (uint32_t n = 0; n < N; n++) {
            const uint64_t i = (uint64_t)g * N + n;
            if (out_hard) out_hard[i] = (r.node_taint_hard[n] & ~r.tolerate_hard[g]) != 0;
            if (out_soft) out_soft[i] = (uint32_t)__builtin_popcountll(r.node_taint_soft[n] & ~r.tolerate_soft[g]);
            bool has_req = false, req_ok = false;
            uint32_t pref = 0;
            for (uint32_t t = 0; t < r.n_terms; t++) {
                if (r.term_owner[t] != (int32_t)g) continue;
                const bool ok = match(t, n);
                if (r.term_weight[t] == 0) {
                    has_req = true;
                    req_ok |= ok;
                } else if (ok) {
                    pref += r.term_weight[t];
                }
            }
            if (out_affinity) out_affinity[i] = !has_req || req_ok;
            if (out_preferred) out_preferred[i] = pref;
        }
    return KS_OK;
}
KSH_CATCH

int ksh_reconcile_nodes(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const int32_t* group, uint32_t n_groups,
                        const char* const* topology_keys, uint32_t K, const uint32_t* max_skew,
                        const uint32_t* min_domains, const char* const* existing_node_names,
                        const uint64_t* existing_offset, const ksh_pod_affinity* aff, const ks_bind_scoring* scoring,
                        const ksh_node_rules* rules, int policy, int32_t* out_status, int32_t* out_node_idx, char* json,
                        size_t cap, int64_t* out_json_off) try {
    if (!scoring) return fail(KS_ERR_INVALID, "NULL scoring");
    const ksh_pod_affinity none{};
    return reconcile_spread(c, pods, n, group, n_groups, topology_keys, K, max_skew, min_domains, existing_node_names,
                            existing_offset, aff ? aff : &none, policy, out_status, out_node_idx, json, cap,
                            out_json_off, {RM_NODES, scoring, rules});
}
KSH_CATCH

int ksh_compile_resources(ksh_context* c, const ks_pod_obj* pods, uint64_t n, char* names, size_t cap,
                          int64_t* out_node_free, int64_t* out_pod_req) try {
    if (!c || (n && !pods) || (cap && !names)) return fail(KS_ERR_INVALID, "NULL argument");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    CompiledResources res;
    const int rc = compile_resources(c, pods, n, &res);
    if (rc) return rc;
    StringList list{names, cap};
    for (const uint32_t id : res.ids)
        if (list.append(c->res_name[id].c_str(), c->res_name[id].size() + 1) < 0)
            return fail(KS_ERR_RANGE, "the resource names do not fit in cap bytes");
    if (out_node_free) std::copy(res.node_free.begin(), res.node_free.end(), out_node_free);
    if (out_pod_req) std::copy(res.pod_req.begin(), res.pod_req.end(), out_pod_req);
    return (int)res.ids.size();
}
KSH_CATCH

int ksh_reconcile_fit(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const int32_t* group, uint32_t n_groups,
                      const char* const* topology_keys, uint32_t K, const uint32_t* max_skew,
                      const uint32_t* min_domains, const char* const* existing_node_names,
                      const uint64_t* existing_offset, const ksh_pod_affinity* aff, const ks_bind_scoring* scoring,
                      const ksh_node_rules* rules, int policy, int32_t* out_status, int32_t* out_node_idx, char* json,
                      size_t cap, int64_t* out_json_off) try {
    if (!scoring) return fail(KS_ERR_INVALID, "NULL scoring");
    const ksh_pod_affinity none{};
    return reconcile_spread(c, pods, n, group, n_groups, topology_keys, K, max_skew, min_domains, existing_node_names,
                            existing_offset, aff ? aff : &none, policy, out_status, out_node_idx, json, cap,
                            out_json_off, {RM_FIT, scoring, rules});
}
KSH_CATCH

int ksh_reconcile_fit_gangs(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const int32_t* group, uint32_t n_groups,
                            const char* const* topology_keys, uint32_t K, const uint32_t* max_skew,
                            const uint32_t* min_domains, const char* const* existing_node_names,
                            const uint64_t* existing_offset, const ksh_pod_affinity* aff,
                            const ks_bind_scoring* scoring, const ksh_node_rules* rules, const uint64_t* gang_offset,
                            uint64_t n_gangs, const uint32_t* min_member, int policy, int32_t* out_status,
                            int32_t* out_node_idx, uint32_t* out_placed, char* json, size_t cap,
                            int64_t* out_json_off) try {
    if (!scoring || !gang_offset) return fail(KS_ERR_INVALID, "NULL scoring or gang_offset");
    const ksh_pod_affinity none{};
    return reconcile_spread(c, pods, n, group, n_groups, topology_keys, K, max_skew, min_domains, existing_node_names,
                            existing_offset, aff ? aff : &none, policy, out_status, out_node_idx, json, cap,
                            out_json_off, {RM_FIT_GANGS, scoring, rules, gang_offset, n_gangs, min_member, out_placed});
}
KSH_CATCH

int ksh_preempt_fit_pods(ksh_context* c, const ks_pod_obj* pods, uint64_t n, const int32_t* group, uint32_t n_groups,
                         const ksh_node_rules* rules, const int32_t* pod_priority, uint32_t max_victims,
                         ks_preemption* out, char* victims, size_t cap, int64_t* out_victim_off) try {
    if (!c || (n && (!pods || !group || !pod_priority || !out))) return fail(KS_ERR_INVALID, "NULL argument");
    if (max_victims == 0 || max_victims > KS_PREEMPT_MAX_VICTIMS)
        return fail(KS_ERR_RANGE, "max_victims must be in [1, " + std::to_string(KS_PREEMPT_MAX_VICTIMS) + "]");
    for (uint64_t i = 0; i < n; i++)
        if (group[i] < -1 || group[i] >= (int64_t)n_groups)
            return fail(KS_ERR_INVALID, "pod " + std::to_string(i) + ": group outside [-1, n_groups)");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    int rc = device_ready(c, ks_fit_preempt, "ks_fit_preempt");
    if (rc) return rc;
    if (out_victim_off)
        for (uint64_t i = 0; i < n; i++) out_victim_off[i] = -1;
    CompiledNodeRules cr;
    rc = compile_node_rules(c, n_groups, rules, &cr);
    if (rc || n == 0) return rc;
    CompiledResources res;
    rc = compile_resources(c, pods, n, &res);
    if (rc) return rc;
    ks_pods kp;
    rc = pack_batch(c, pods, n, &kp); // after this the device's free[] comes from the bound rows below
    if (rc) return rc;
    const size_t B = c->bnode.size(), R = res.ids.size();
    std::vector<int32_t> col(c->res_name.size(), -1);
    for (size_t r = 0; r < R; r++) col[res.ids[r]] = (int32_t)r;
    std::vector<int32_t> prio(B);
    std::vector<int64_t> breq(B * R, 0);
    for (size_t b = 0; b < B; b++) {
        prio[b] = c->blen[b] ? c->bprio[b] : INT32_MAX; // anonymous: cannot be evicted
        breq[b * R] = 1;
        for (const ExtQty& e : c->bext[b]) // malformed requested quantities were reported by compile_resources
            if (e.res < col.size() && col[e.res] > 0) breq[b * R + (size_t)col[e.res]] = e.v;
    }
    std::vector<int32_t> vic((size_t)n * max_victims);
    const ks_bound_pods kb{B, c->bnode.data(), c->bcpu.data(), c->bmem.data(), prio.data()};
    const ks_bind_resources br{(uint32_t)R, res.node_free.data(), res.pod_req.data()};
    rc = ks_fit_preempt(c->snap, &kp, group, n_groups, &cr.r, &br, pod_priority, &kb, breq.data(), max_victims, out,
                        vic.data(), nullptr);
    if (rc || !victims || !out_victim_off) return rc;
    StringList list{victims, cap};
    std::string keys;
    for (uint64_t i = 0; i < n; i++) {
        if (out[i].node_idx < 0) continue;
        keys.clear();
        for (uint32_t j = 0; j < out[i].n_victims; j++) { // "namespace/name", NUL-terminated, in visit order
            const size_t b = (size_t)vic[(size_t)i * max_victims + j];
            keys.append(c->bkeys.data() + c->boff[b], c->blen[b]);
            keys.push_back('\0');
        }
        out_victim_off[i] = list.append(keys.data(), keys.size());
    }
    return KS_OK;
}
KSH_CATCH

// ksh_drain_nodes' candidates under the full filter: the context's taints and the groups' rules compiled as
// ksh_preempt_fit_pods compiles them, and the batch's resources (the pod count always among them) from the drained
// pods.  Those pods are bound to their candidate, which is never a destination, so the context's node_free is used as
// it is.
int ksh_drain_fit_nodes(ksh_context* c, const char* const* node_names, uint64_t n, const ks_pod_obj* pods,
                        const uint64_t* pod_offset, const int32_t* group, uint32_t n_groups, const ksh_node_rules* rules,
                        int policy, uint32_t flags, uint32_t* out_placed, int32_t* out_node_idx,
                        uint32_t* out_refused) try {
    if (!c || !pod_offset || (n && (!node_names || !out_placed))) return fail(KS_ERR_INVALID, "NULL argument");
    if (pod_offset[0] != 0) return fail(KS_ERR_INVALID, "pod_offset[0] must be 0");
    for (uint64_t d = 0; d < n; d++)
        if (pod_offset[d + 1] < pod_offset[d]) return fail(KS_ERR_INVALID, "pod offsets decrease");
    const uint64_t P = pod_offset[n];
    if (P && (!pods || !out_node_idx || !group)) return fail(KS_ERR_INVALID, "NULL argument");
    for (uint64_t i = 0; i < P; i++)
        if (group[i] < -1 || group[i] >= (int64_t)n_groups)
            return fail(KS_ERR_INVALID, "pod " + std::to_string(i) + ": group outside [-1, n_groups)");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    std::vector<int32_t> node(n);
    for (uint64_t d = 0; d < n; d++) { // mis-grouped input is refused before anything is packed
        const char* name = node_names[d];
        if (!name) return fail(KS_ERR_INVALID, "candidate " + std::to_string(d) + ": node name is NULL");
        node[d] = node_index_of(c, name);
        if (node[d] < 0) return fail(KS_ERR_INVALID, "candidate " + std::to_string(d) + ": node \"" + name + "\" is not in the store");
        for (uint64_t i = pod_offset[d]; i < pod_offset[d + 1]; i++)
            if (!ksh_is_pod_bound(&pods[i]) || std::strcmp(pods[i].node_name, name) != 0)
                return fail(KS_ERR_INVALID, "pod " + std::to_string(i) + " (" + nz(pods[i].ns) + "/" + nz(pods[i].name) +
                                                ") has spec.nodeName \"" + (ksh_is_pod_bound(&pods[i]) ? pods[i].node_name : "") +
                                                "\", not its candidate's node \"" + name + "\"");
    }
    int rc = device_ready(c, ks_fit_drain_check, "ks_fit_drain_check");
    if (rc) return rc;
    CompiledNodeRules cr;
    rc = compile_node_rules(c, n_groups, rules, &cr);
    if (rc) return rc;
    CompiledResources res;
    rc = compile_resources(c, pods, P, &res);
    if (rc) return rc;
    ks_pods kp;
    rc = pack_batch(c, pods, P, &kp);
    if (rc) return rc;
    const ks_drain_candidates kc{n, node.data(), pod_offset};
    const ks_bind_resources br{(uint32_t)res.ids.size(), res.node_free.data(), res.pod_req.data()};
    return ks_fit_drain_check(c->snap, &kp, group, n_groups, &cr.r, &br, &kc, policy, flags, out_placed, out_node_idx,
                              nullptr, out_refused);
}
KSH_CATCH

// ksh_scaleup_estimate's objects, packed for ks_scaleup_estimate: the templates (names, allocatable as
// ksh_context_set_nodes parses it, capacity = allocatable minus the overhead pods), the pending pods' requests, and the
// call-local label dictionary.  ksh_scaleup_fit_estimate packs its objects the same way.
struct ScaleupObjects {
    std::unordered_map<std::string, uint32_t> index; // template name -> template
    std::vector<int64_t> ac, am, fc, fm, rc, rm;
    std::vector<uint64_t> lab, sel;
    uint32_t W = 1;
};

static int scaleup_objects(const ks_node_obj* templates, uint64_t n_templates, const ks_pod_obj* overhead_pods,
                           uint64_t n_overhead, const ks_pod_obj* pods, uint64_t n_pods, ScaleupObjects* o) {
    o->ac.resize(n_templates);
    o->am.resize(n_templates);
    o->fc.resize(n_templates);
    o->fm.resize(n_templates);
    for (uint64_t t = 0; t < n_templates; t++) {
        if (!templates[t].name) return fail(KS_ERR_INVALID, "template " + std::to_string(t) + ": name is NULL");
        if (!o->index.emplace(templates[t].name, (uint32_t)t).second)
            return fail(KS_ERR_INVALID, "template " + std::to_string(t) + ": duplicate name \"" + templates[t].name + "\"");
        std::string err;
        const int rc = parse_node_allocatable(templates[t], &o->ac[t], &o->am[t], &err);
        if (rc) return fail(rc, "template " + std::to_string(t) + ": " + err);
        o->fc[t] = o->ac[t];
        o->fm[t] = o->am[t];
    }
    for (uint64_t i = 0; i < n_overhead; i++) { // DaemonSet pods, charged to the template spec.nodeName names
        const ks_pod_obj& pod = overhead_pods[i];
        const std::string who = "overhead pod " + std::to_string(i) + " (" + nz(pod.ns) + "/" + nz(pod.name) + ")";
        if (!ksh_is_pod_bound(&pod)) return fail(KS_ERR_INVALID, who + " has no spec.nodeName naming its template");
        const auto it = o->index.find(pod.node_name);
        if (it == o->index.end()) return fail(KS_ERR_INVALID, who + " names unknown template \"" + pod.node_name + "\"");
        int64_t cpu, mem;
        std::string err;
        const int rc = total_pod_resources(&pod, &cpu, &mem, &err);
        if (rc) return fail(rc, who + ": " + err);
        if (__builtin_sub_overflow(o->fc[it->second], cpu, &o->fc[it->second]) ||
            __builtin_sub_overflow(o->fm[it->second], mem, &o->fm[it->second]))
            return fail(KS_ERR_RANGE, who + ": capacity of its template overflows");
    }
    // pending pods: unbound, requests as ksh_select_nodes packs them
    o->rc.resize(n_pods);
    o->rm.resize(n_pods);
    for (uint64_t p = 0; p < n_pods; p++) {
        const std::string who = "pod " + std::to_string(p) + " (" + nz(pods[p].ns) + "/" + nz(pods[p].name) + ")";
        if (ksh_is_pod_bound(&pods[p]))
            return fail(KS_ERR_INVALID, who + " has spec.nodeName \"" + pods[p].node_name + "\": not a pending pod");
        std::string err;
        const int rc = total_pod_resources(&pods[p], &o->rc[p], &o->rm[p], &err);
        if (rc) return fail(rc, who + ": " + err);
    }
    // call-local dictionary: a bit for every pair that some pending pod names and some template carries, in the order
    // the pods name them; every other selector pair takes the never-set bit (the last bit of the last word)
    std::unordered_map<std::string, int32_t> carried; // "key\0value" -> bit, -1 until a pod names it
    for (uint64_t t = 0; t < n_templates; t++)
        if (templates[t].has_labels)
            for (uint32_t i = 0; i < templates[t].n_labels; i++)
                carried.emplace(std::string(nz(templates[t].labels[i].key)) + '\0' + nz(templates[t].labels[i].val), -1);
    uint32_t bits = 0;
    for (uint64_t p = 0; p < n_pods; p++) {
        if (!(pods[p].has_spec && pods[p].has_node_selector)) continue;
        for (uint32_t i = 0; i < pods[p].n_selector; i++) {
            const auto it = carried.find(std::string(nz(pods[p].selector[i].key)) + '\0' + nz(pods[p].selector[i].val));
            if (it != carried.end() && it->second < 0) it->second = (int32_t)bits++;
        }
    }
    if (bits > 64 * KS_MAX_LABEL_WORDS - 1)
        return fail(KS_ERR_RANGE, "more than 511 distinct (key,value) pairs named by pending pods and carried by templates");
    const uint32_t W = words_for_bits(bits), never = 64 * W - 1;
    o->W = W;
    o->lab.assign(n_templates * W, 0);
    o->sel.assign(n_pods * W, 0);
    for (uint64_t t = 0; t < n_templates; t++)
        if (templates[t].has_labels)
            for (uint32_t i = 0; i < templates[t].n_labels; i++) {
                const int32_t b = carried[std::string(nz(templates[t].labels[i].key)) + '\0' + nz(templates[t].labels[i].val)];
                if (b >= 0) o->lab[t * W + b / 64] |= 1ull << (b % 64);
            }
    for (uint64_t p = 0; p < n_pods; p++) {
        if (!(pods[p].has_spec && pods[p].has_node_selector)) continue;
        for (uint32_t i = 0; i < pods[p].n_selector; i++) {
            const auto it = carried.find(std::string(nz(pods[p].selector[i].key)) + '\0' + nz(pods[p].selector[i].val));
            const uint32_t b = it != carried.end() ? (uint32_t)it->second : never;
            o->sel[p * W + b / 64] |= 1ull << (b % 64);
        }
    }
    return KS_OK;
}

int ksh_scaleup_estimate(ksh_context* c, const ks_node_obj* templates, uint64_t n_templates, const uint32_t* max_nodes,
                         const ks_pod_obj* overhead_pods, uint64_t n_overhead, const ks_pod_obj* pods, uint64_t n_pods,
                         ks_scaleup_option* out, int32_t* out_best, int32_t* out_node, ks_pod_reasons* out_reasons) try {
    if (!c || !out_best || (n_templates && (!templates || !max_nodes || !out)) || (n_overhead && !overhead_pods) ||
        (n_pods && !pods))
        return fail(KS_ERR_INVALID, "NULL argument");
    if (n_pods > KS_SCALEUP_MAX_PODS || n_templates > KS_SCALEUP_MAX_TEMPLATES)
        return fail(KS_ERR_RANGE, "more than " + std::to_string(KS_SCALEUP_MAX_PODS) + " pods or " +
                                      std::to_string(KS_SCALEUP_MAX_TEMPLATES) + " templates");
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    ScaleupObjects o;
    int rc = scaleup_objects(templates, n_templates, overhead_pods, n_overhead, pods, n_pods, &o);
    if (rc) return rc;
    rc = device_ready(c, ks_scaleup_estimate, "ks_scaleup_estimate");
    if (rc) return rc;
    ks_pods kp{n_pods, o.rc.data(), o.rm.data(), o.sel.data(), KS_MEM_HOST};
    ks_node_templates kt{n_templates, o.W, o.ac.data(), o.am.data(), o.fc.data(), o.fm.data(), o.lab.data(), max_nodes};
    return ks_scaleup_estimate(c->snap, &kp, &kt, out, out_best, out_node, out_reasons);
}
KSH_CATCH

// ksh_scaleup_estimate's objects under the full filter: the templates' taints and label values as the node side of the
// rule compilation, and the batch's resources with each template's node_free from its allocatable and overhead pods
int ksh_scaleup_fit_estimate(ksh_context* c, const ks_node_obj* templates, uint64_t n_templates, const uint32_t* max_nodes,
                             const uint64_t* template_taint_offset, const ksh_taint* template_taints,
                             const ks_pod_obj* overhead_pods, uint64_t n_overhead, const ks_pod_obj* pods,
                             uint64_t n_pods, const int32_t* group, uint32_t n_groups, const ksh_node_rules* rules,
                             ks_scaleup_option* out, int32_t* out_best, int32_t* out_node, uint32_t* out_refused) try {
    if (!c || !out_best || (n_templates && (!templates || !max_nodes || !out)) || (n_overhead && !overhead_pods) ||
        (n_pods && (!pods || !group)))
        return fail(KS_ERR_INVALID, "NULL argument");
    if (n_pods > KS_SCALEUP_MAX_PODS || n_templates > KS_SCALEUP_MAX_TEMPLATES)
        return fail(KS_ERR_RANGE, "more than " + std::to_string(KS_SCALEUP_MAX_PODS) + " pods or " +
                                      std::to_string(KS_SCALEUP_MAX_TEMPLATES) + " templates");
    for (uint64_t i = 0; i < n_pods; i++)
        if (group[i] < -1 || group[i] >= (int64_t)n_groups)
            return fail(KS_ERR_INVALID, "pod " + std::to_string(i) + ": group outside [-1, n_groups)");
    const uint64_t* toff = template_taint_offset;
    if (toff && toff[n_templates] && !template_taints) return fail(KS_ERR_INVALID, "NULL template_taints");
    // the templates' taints, checked as ksh_context_set_node_taints checks a node's
    std::vector<std::vector<Taint>> taints(n_templates);
    for (uint64_t t = 0; toff && t < n_templates; t++) {
        if (toff[t + 1] < toff[t]) return fail(KS_ERR_INVALID, "template taint offsets decrease");
        for (uint64_t i = toff[t]; i < toff[t + 1]; i++) {
            const std::string e = nz(template_taints[i].effect);
            if (!template_taints[i].key || !*template_taints[i].key ||
                (e != "NoSchedule" && e != "PreferNoSchedule" && e != "NoExecute"))
                return fail(KS_ERR_INVALID, "template taint " + std::to_string(i) + ": empty key or effect \"" + e + "\"");
            taints[t].push_back({template_taints[i].key, nz(template_taints[i].value), e});
        }
    }
    std::lock_guard<std::recursive_mutex> lk(c->mu);
    ScaleupObjects o;
    int rc = scaleup_objects(templates, n_templates, overhead_pods, n_overhead, pods, n_pods, &o);
    if (rc) return rc;
    // the rules over the templates: their taints, and each rule key's values numbered in template order
    RuleNodes nodes;
    nodes.N = (uint32_t)n_templates;
    nodes.what = "the templates";
    nodes.taints_of = [&](uint32_t t) { return &taints[t]; };
    nodes.domains = [&](const std::string& key, int32_t* dom, std::vector<std::string>* values) {
        std::unordered_map<std::string, int32_t> of_value;
        for (uint64_t t = 0; t < n_templates; t++) {
            dom[t] = -1;
            for (uint32_t i = 0; templates[t].has_labels && i < templates[t].n_labels; i++) {
                if (key != nz(templates[t].labels[i].key)) continue;
                const auto it = of_value.emplace(nz(templates[t].labels[i].val), (int32_t)values->size()).first;
                if (it->second == (int32_t)values->size()) values->push_back(it->first);
                dom[t] = it->second;
                break; // the first of a repeated key, as the store keeps it
            }
        }
    };
    CompiledNodeRules cr;
    rc = compile_rules_over(nodes, n_groups, rules, &cr);
    if (rc) return rc;
    // resources: the batch's names; node_free = a template's allocatable of each (0 when missing) minus its overhead
    // pods' requests, and for "pods" minus their number
    CompiledResources res;
    rc = batch_resources(c, pods, n_pods, &res);
    if (rc) return rc;
    const size_t R = res.ids.size(), T = n_templates;
    std::vector<int32_t> col(c->res_name.size(), -1);
    for (size_t r = 0; r < R; r++) col[res.ids[r]] = (int32_t)r;
    res.node_free.assign(R * T, 0);
    for (size_t t = 0; t < T; t++)
        for (const ExtQty& e : node_ext(c, templates[t])) {
            if (e.res >= col.size() || col[e.res] < 0) continue;
            if (e.err) return ext_error(c, "template '" + std::string(templates[t].name) + "'", "allocatable ", e);
            res.node_free[(size_t)col[e.res] * T + t] = e.v;
        }
    for (uint64_t i = 0; i < n_overhead; i++) {
        const size_t t = o.index[overhead_pods[i].node_name]; // checked by scaleup_objects
        bool over = __builtin_sub_overflow(res.node_free[t], 1, &res.node_free[t]);
        for (const ExtQty& e : pod_ext(c, &overhead_pods[i])) {
            if (e.res >= col.size() || col[e.res] <= 0) continue;
            if (e.err) return ext_error(c, "overhead pod '" + pod_key(&overhead_pods[i]) + "'", "request of ", e);
            int64_t& f = res.node_free[(size_t)col[e.res] * T + t];
            over |= __builtin_sub_overflow(f, e.v, &f);
        }
        if (over) return fail(KS_ERR_RANGE, "free resources of a template overflow int64");
    }
    rc = device_ready(c, ks_fit_scaleup_estimate, "ks_fit_scaleup_estimate");
    if (rc) return rc;
    ks_pods kp{n_pods, o.rc.data(), o.rm.data(), o.sel.data(), KS_MEM_HOST};
    ks_node_templates kt{n_templates, o.W, o.ac.data(), o.am.data(), o.fc.data(), o.fm.data(), o.lab.data(), max_nodes};
    const ks_bind_resources br{(uint32_t)R, res.node_free.data(), res.pod_req.data()};
    return ks_fit_scaleup_estimate(c->snap, &kp, group, n_groups, &cr.r, &br, &kt, out, out_best, out_node, out_refused,
                                   nullptr);
}
KSH_CATCH

} // extern "C"
