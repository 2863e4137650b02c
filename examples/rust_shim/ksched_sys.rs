// ksched_sys.rs — `extern "C"` binding of libksched.so for the reference's Rust host (SURVEY.md §8(b), §8(f)#4).
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no rustc/cargo and the reference's 229 crates are not
// vendored.  Hand-written from include/ksched.h, include/ksched_host.h and include/ks_objects.h (bindgen over those
// headers produces the same items); tests/test_abi.py keeps this file honest by checking that every function declared
// here is exported by libksched.so, and the same ABI is driven from C by examples/reconcile_loop.c and from Python by
// kube-scheduler-rs-reference_b200/_capi.py + host.py.
//
// Drop into the reference as src/ksched_sys.rs (`mod ksched_sys;` in src/main.rs) together with src/ksched.rs
// (the safe wrapper next to this file).  build.rs:
//     println!("cargo:rustc-link-search=native=/opt/ksched/lib");
//     println!("cargo:rustc-link-lib=dylib=ksched");
#![allow(non_camel_case_types, dead_code)]
use std::os::raw::{c_char, c_int, c_void};

pub const KS_OK: c_int = 0;
pub const KS_SCORE_LEFTOVER: c_int = 0;
pub const KS_SCORE_LEAST_ALLOCATED: c_int = 1;
/// Bin-packing (upstream MostAllocated); 2 is reserved and rejected.
pub const KS_SCORE_MOST_ALLOCATED: c_int = 3;
/// Upstream's default profile: LeastAllocated + BalancedAllocation, in [0, 200].
pub const KS_SCORE_LEAST_BALANCED: c_int = 4;
pub const KS_MEM_HOST: i32 = 0;
pub const KS_MEM_DEVICE: i32 = 1;
pub const KS_ERR_INVALID: c_int = -1; // a NULL or malformed argument
pub const KS_ERR_NO_DEVICE: c_int = -8; // packing-only context or no CUDA device
pub const KS_CELL_OK: c_int = 0;
pub const KS_CELL_NOT_ENOUGH_RESOURCES: c_int = 1; // InvalidNodeReason::NotEnoughResources  (src/predicates.rs:16)
pub const KS_CELL_NODE_SELECTOR_MISMATCH: c_int = 2; // InvalidNodeReason::NodeSelectorMismatch (src/predicates.rs:17)
pub const KSH_RECONCILE_OK: c_int = 0;
pub const KSH_RECONCILE_NO_NODE_FOUND: c_int = 1; // ReconcileError::NoNodeFound (src/error.rs)
pub const KSH_RECONCILE_BINDING_OBJECT_FAILED: c_int = 2; // ReconcileError::CreateBindingObjectFailed
pub const KSH_RECONCILE_GANG_UNSATISFIED: c_int = 4; // ksh_reconcile_gangs: the pod's group rolled back
pub const KSH_RECONCILE_SPREAD_UNSATISFIED: c_int = 5; // ksh_reconcile_spread: spread constraints refused every node
pub const KSH_RECONCILE_AFFINITY_UNSATISFIED: c_int = 6; // ksh_reconcile_affinity: pod (anti-)affinity refused every node
pub const KSH_RECONCILE_NODE_RULES_UNSATISFIED: c_int = 7; // ksh_reconcile_nodes: taints or node affinity refused every node
pub const KSH_RECONCILE_INSUFFICIENT_RESOURCES: c_int = 8; // ksh_reconcile_fit: every node that fit lacked a resource
pub const KS_REFERENCE_ATTEMPTS: u32 = 5; // ATTEMPTS, src/main.rs:49
pub const KS_MAX_PEERS: usize = 15;
pub const KS_TOPK_MAX: u32 = 32; // largest k of ks_select_topk / ksh_rank_nodes
pub const KS_PREEMPT_MAX_VICTIMS: u32 = 128; // largest max_victims of ks_preempt / ksh_preempt_pods
pub const KS_GANG_MAX_SIZE: u32 = 1024; // most pods in one group of ks_gang_bind / ksh_reconcile_gangs
pub const KS_DRAIN_MAX_PODS: u32 = 1024; // most pods of one candidate of ks_drain_check / ksh_drain_nodes
pub const KS_DRAIN_EXCLUDE_CANDIDATES: u32 = 1; // no candidate's node is a destination of any candidate
pub const KS_SCALEUP_MAX_NODES: u32 = 1024; // most new nodes of one template of ks_scaleup_estimate
pub const KS_SCALEUP_MAX_PODS: u32 = 65536; // most pods of one ks_scaleup_estimate call
pub const KS_SCALEUP_MAX_TEMPLATES: u32 = 4096; // most templates of one ks_scaleup_estimate call
pub const KS_REPLICAS_MAX_SPECS: u32 = 4096; // most specs of one ks_place_replicas call
pub const KS_REPLICAS_MAX: u32 = 65536; // most copies of one spec
pub const KS_REPLICAS_MAX_TOTAL: u32 = 1 << 24; // most copies of one ks_place_replicas call
pub const KS_SPREAD_MAX_DOMAINS: u32 = 1 << 20; // most topology domains of one ks_place_replicas_spread call
pub const KS_SPREAD_MAX_EXISTING: u32 = 1 << 24; // most existing pods counted in one domain
pub const KS_SPREAD_MAX_COUNTS: u64 = 1 << 26; // most specs x domains of existing or output counts
pub const KS_SPREAD_MAX_KEYS: u32 = 4; // most topology keys of one ks_place_replicas_spread_multi call
pub const KS_SPREAD_BIND_MAX_PODS: u32 = 65536; // most pods of one ks_spread_bind call
pub const KS_SPREAD_BIND_MAX_GROUPS: u32 = 4096; // most groups of one ks_spread_bind call
pub const KS_POD_AFFINITY: u8 = 0; // ks_pod_affinity term kinds
pub const KS_POD_ANTI_AFFINITY: u8 = 1;
pub const KS_AFFINITY_MAX_TERMS: u32 = 16384; // most terms of one ks_affinity_bind call
pub const KS_AFFINITY_MAX_TARGETS: u64 = 1 << 22; // most target entries over all terms
pub const KS_AFFINITY_MAX_EXISTING: u64 = 1 << 24; // most existing pods
pub const KS_AFFINITY_MAX_UPDATES: u64 = 1 << 24; // most compiled update entries
pub const KS_POD_AFFINITY_PREFERRED: u8 = 2; // ks_profile_bind: preferred terms score only
pub const KS_POD_ANTI_AFFINITY_PREFERRED: u8 = 3;
pub const KS_NODE_RULES_MAX_TAINTS: u32 = 64; // ks_node_bind
pub const KS_NODE_RULES_MAX_KEYS: usize = 16;
pub const KS_NODE_RULES_MAX_PREFERRED: u32 = 4096;
pub const KS_NODE_RULES_MAX_WORDS: u64 = 1 << 26;
pub const KS_BIND_MAX_RESOURCES: u32 = 8; // ks_fit_bind: most scalar resources of one call

#[repr(C)]
pub struct ks_kv {
    pub key: *const c_char,
    pub val: *const c_char,
}
#[repr(C)]
pub struct ks_container_obj {
    pub has_requests: i32,
    pub n_requests: u32,
    pub requests: *const ks_kv,
}
#[repr(C)]
pub struct ks_pod_obj {
    pub ns: *const c_char,
    pub name: *const c_char,
    pub has_spec: i32,
    pub node_name: *const c_char,
    pub n_containers: u32,
    pub containers: *const ks_container_obj,
    pub has_node_selector: i32,
    pub n_selector: u32,
    pub selector: *const ks_kv,
    pub metadata_json: *const c_char, // serde_json::to_string(&pod.metadata): emitted verbatim in the Binding (src/main.rs:88)
}
#[repr(C)]
pub struct ks_node_obj {
    pub name: *const c_char,
    pub has_labels: i32,
    pub n_labels: u32,
    pub labels: *const ks_kv,
    pub has_allocatable: i32,
    pub n_allocatable: u32,
    pub allocatable: *const ks_kv,
}
#[repr(C)]
pub struct ks_pods {
    pub n: u64,
    pub req_cpu: *const i64,
    pub req_mem: *const i64,
    pub sel: *const u64,
    pub mem_space: i32,
}
#[repr(C)]
pub struct ks_exchange {
    pub world: u32,
    pub rank: u32,
    pub n_peers: u32,
    pub peer_node_idx: [*mut i32; KS_MAX_PEERS],
    pub peer_score: [*mut i64; KS_MAX_PEERS],
    pub peer_flag: [*mut u32; KS_MAX_PEERS],
    pub local_flags: *mut u32,
    pub local_state: *mut u32,
}
#[repr(C)]
pub struct ks_bindings {
    pub node_idx: *mut i32,
    pub score: *mut i64,
    pub feasible_cnt: *mut u32,
    pub mem_space: i32,
    pub mask: *mut u8,
    pub mask_row_bytes: u64,
    pub mask_space: i32,
    pub bindings_ready_event: *mut c_void, // optional cudaEvent_t
    pub exchange: *const ks_exchange,      // optional fused all-gather over NVLink
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct ks_pod_reasons {
    pub insufficient_cpu: u32,
    pub insufficient_memory: u32,
    pub not_enough_resources: u32,
    pub node_selector_mismatch: u32,
}
#[repr(C)]
pub struct ks_bound_pods {
    pub n: u64,
    pub node_idx: *const i32,
    pub req_cpu: *const i64,
    pub req_mem: *const i64,
    pub priority: *const i32,
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct ks_preemption {
    pub node_idx: i32,
    pub n_victims: u32,
    pub candidates: u32,
    pub feasible_cnt: u32,
    pub max_victim_priority: i32,
    pub reserved: u32,
    pub victim_priority_sum: i64,
}
#[repr(C)]
pub struct ks_gangs {
    pub n: u64,
    pub offset: *const u64,
    pub min_member: *const u32,
}
#[repr(C)]
pub struct ks_drain_candidates {
    pub n: u64,
    pub node_idx: *const i32,
    pub offset: *const u64,
}
#[repr(C)]
pub struct ks_node_templates {
    pub n: u64,
    pub label_words: u32,
    pub alloc_cpu: *const i64,
    pub alloc_mem: *const i64,
    pub free_cpu: *const i64,
    pub free_mem: *const i64,
    pub labels: *const u64,
    pub max_nodes: *const u32,
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct ks_scaleup_option {
    pub nodes: u32,
    pub placed: u32,
    pub eligible: u32,
    pub utilization: i32,
    pub used_cpu: i64,
    pub used_mem: i64,
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct ks_replica_plan {
    pub capacity: u64,
    pub placed: u32,
    pub nodes: u32,
    pub feasible_cnt: u32,
    pub max_per_node: u32,
    pub last_score: i64,
}
#[repr(C)]
pub struct ks_spread {
    pub n_domains: u32,
    pub node_domain: *const i32,
    pub max_skew: *const u32,
    pub min_domains: *const u32,
    pub existing: *const u32,
}
#[repr(C)]
pub struct ks_spread_multi {
    pub n_keys: u32,
    pub n_domains: [u32; KS_SPREAD_MAX_KEYS as usize],
    pub node_domain: [*const i32; KS_SPREAD_MAX_KEYS as usize],
    pub max_skew: *const u32,
    pub min_domains: *const u32,
    pub existing: *const u32,
}
#[repr(C)]
pub struct ks_pod_affinity {
    pub n_terms: u32,
    pub owner: *const i32,
    pub kind: *const u8,
    pub key: *const u32,
    pub target_offset: *const u64,
    pub target: *const i32,
    pub n_existing: u64,
    pub existing_group: *const i32,
    pub existing_node: *const i32,
}
#[repr(C)]
pub struct ks_bind_scoring {
    pub soft_skew: *const u32,
    pub soft_all_keys: *const u8,
    pub term_weight: *const u32,
    pub hard_affinity_weight: u32,
    pub weight_spread: u32,
    pub weight_affinity: u32,
}
#[repr(C)]
pub struct ks_node_rules {
    pub n_taints: u32,
    pub node_taint_hard: *const u64,
    pub node_taint_soft: *const u64,
    pub tolerate_hard: *const u64,
    pub tolerate_soft: *const u64,
    pub n_keys: u32,
    pub n_domains: [u32; KS_NODE_RULES_MAX_KEYS],
    pub node_domain: [*const i32; KS_NODE_RULES_MAX_KEYS],
    pub n_exprs: u32,
    pub expr_key: *const u32,
    pub expr_set_offset: *const u64,
    pub expr_set: *const u64,
    pub n_terms: u32,
    pub term_owner: *const i32,
    pub term_weight: *const u32,
    pub term_expr_offset: *const u32,
    pub weight_taint: u32,
    pub weight_node_affinity: u32,
}
#[repr(C)]
pub struct ks_bind_resources {
    pub n_res: u32,
    pub node_free: *const i64,
    pub pod_req: *const i64,
}
#[repr(C)]
pub struct ksh_taint {
    pub key: *const c_char,
    pub value: *const c_char,
    pub effect: *const c_char,
}
#[repr(C)]
pub struct ksh_toleration {
    pub key: *const c_char,
    pub op: *const c_char,
    pub value: *const c_char,
    pub effect: *const c_char,
}
#[repr(C)]
pub struct ksh_node_selector_requirement {
    pub key: *const c_char,
    pub op: *const c_char,
    pub values: *const *const c_char,
    pub n_values: u32,
}
#[repr(C)]
pub struct ksh_node_rules {
    pub toleration_offset: *const u64,
    pub tolerations: *const ksh_toleration,
    pub n_terms: u32,
    pub term_owner: *const i32,
    pub term_weight: *const u32,
    pub term_req_offset: *const u64,
    pub requirements: *const ksh_node_selector_requirement,
    pub weight_taint: u32,
    pub weight_node_affinity: u32,
}
#[repr(C)]
pub struct ksh_pod_affinity {
    pub n_terms: u32,
    pub owner: *const i32,
    pub kind: *const u8,
    pub key: *const u32,
    pub target_offset: *const u64,
    pub target: *const i32,
    pub n_existing: u64,
    pub existing_group: *const i32,
    pub existing_node_name: *const *const c_char,
}
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct ks_spread_plan {
    pub placed: u32,
    pub nodes: u32,
    pub max_per_node: u32,
    pub eligible_domains: u32,
    pub min_count: u32,
    pub blocked_domain: i32,
    pub last_score: i64,
}
pub enum ks_snapshot {}
pub enum ks_stream {}
pub enum ksh_context {}

extern "C" {
    pub fn ks_last_error() -> *const c_char;
    pub fn ks_version() -> c_int;
    pub fn ks_device_count() -> c_int;
    pub fn ks_mask_row_bytes(n_nodes: u32) -> u64;
    // ---- packed core (include/ksched.h) ----
    pub fn ks_snapshot_create(device: c_int, out: *mut *mut ks_snapshot) -> c_int;
    pub fn ks_snapshot_destroy(s: *mut ks_snapshot);
    pub fn ks_snapshot_set_nodes(s: *mut ks_snapshot, n: u32, w: u32, cpu: *const i64, mem: *const i64, labels: *const u64) -> c_int;
    pub fn ks_snapshot_set_bound(s: *mut ks_snapshot, b: u64, node: *const i32, cpu: *const i64, mem: *const i64) -> c_int;
    pub fn ks_snapshot_apply_bind(s: *mut ks_snapshot, node: i32, cpu: i64, mem: i64) -> c_int;
    pub fn ks_snapshot_get_free(s: *mut ks_snapshot, cpu: *mut i64, mem: *mut i64) -> c_int;
    pub fn ks_check_cell(s: *mut ks_snapshot, cpu: i64, mem: i64, sel: *const u64, node: u32) -> c_int;
    pub fn ks_check_cells(s: *mut ks_snapshot, pods: *const ks_pods, codes: *mut u8) -> c_int;
    pub fn ks_select(s: *mut ks_snapshot, pods: *const ks_pods, policy: c_int, flags: u32, out: *mut ks_bindings, stream: *mut c_void) -> c_int;
    pub fn ks_select_sampling(s: *mut ks_snapshot, pods: *const ks_pods, attempts: u32, seed: u64, first_pod_index: u64,
                              node_idx: *mut i32, attempts_used: *mut u32, draw_node: *mut i32, draw_code: *mut u8) -> c_int;
    pub fn ks_explain(s: *mut ks_snapshot, pods: *const ks_pods, out: *mut ks_pod_reasons, out_space: i32, stream: *mut c_void) -> c_int;
    pub fn ks_select_topk(s: *mut ks_snapshot, pods: *const ks_pods, policy: c_int, k: u32, node_idx: *mut i32, score: *mut i64,
                          feasible_cnt: *mut u32, out_space: i32, stream: *mut c_void) -> c_int;
    pub fn ks_preempt(s: *mut ks_snapshot, pods: *const ks_pods, pod_priority: *const i32, bound: *const ks_bound_pods,
                      max_victims: u32, out: *mut ks_preemption, out_victims: *mut i32, out_space: i32,
                      stream: *mut c_void) -> c_int;
    pub fn ks_snapshot_commit_claims(s: *mut ks_snapshot, n: u64, node: *const i32, cpu: *const i64, mem: *const i64, accepted: *mut u8) -> c_int;
    pub fn ks_stream_bind(s: *mut ks_snapshot, pods: *const ks_pods, policy: c_int, node_idx: *mut i32, score: *mut i64, rounds: *mut u32) -> c_int;
    pub fn ks_gang_bind(s: *mut ks_snapshot, pods: *const ks_pods, gangs: *const ks_gangs, policy: c_int, node_idx: *mut i32,
                        score: *mut i64, placed: *mut u32, rounds: *mut u32) -> c_int;
    pub fn ks_drain_check(s: *mut ks_snapshot, pods: *const ks_pods, cand: *const ks_drain_candidates, policy: c_int,
                          flags: u32, placed: *mut u32, node_idx: *mut i32, score: *mut i64) -> c_int;
    pub fn ks_scaleup_estimate(s: *mut ks_snapshot, pods: *const ks_pods, t: *const ks_node_templates,
                               out: *mut ks_scaleup_option, best: *mut i32, node: *mut i32,
                               reasons: *mut ks_pod_reasons) -> c_int;
    pub fn ks_place_replicas(s: *mut ks_snapshot, specs: *const ks_pods, replicas: *const u32, policy: c_int,
                             out: *mut ks_replica_plan, node: *mut i32, score: *mut i64) -> c_int;
    pub fn ks_place_replicas_spread(s: *mut ks_snapshot, specs: *const ks_pods, replicas: *const u32, spread: *const ks_spread,
                                    policy: c_int, out: *mut ks_spread_plan, node: *mut i32, score: *mut i64,
                                    domain_count: *mut u32) -> c_int;
    pub fn ks_place_replicas_spread_multi(s: *mut ks_snapshot, specs: *const ks_pods, replicas: *const u32,
                                          spread: *const ks_spread_multi, policy: c_int, out: *mut ks_spread_plan,
                                          node: *mut i32, score: *mut i64, domain_count: *mut u32) -> c_int;
    pub fn ks_spread_bind(s: *mut ks_snapshot, pods: *const ks_pods, group: *const i32, n_groups: u32,
                          spread: *const ks_spread_multi, policy: c_int, node_idx: *mut i32, score: *mut i64,
                          refused: *mut u32, domain_count: *mut u32) -> c_int;
    pub fn ks_affinity_bind(s: *mut ks_snapshot, pods: *const ks_pods, group: *const i32, n_groups: u32,
                            topo: *const ks_spread_multi, aff: *const ks_pod_affinity, policy: c_int,
                            node_idx: *mut i32, score: *mut i64, refused: *mut u32, domain_count: *mut u32) -> c_int;
    pub fn ks_profile_bind(s: *mut ks_snapshot, pods: *const ks_pods, group: *const i32, n_groups: u32,
                           topo: *const ks_spread_multi, aff: *const ks_pod_affinity, scoring: *const ks_bind_scoring,
                           policy: c_int, node_idx: *mut i32, score: *mut i64, parts: *mut i64, refused: *mut u32,
                           domain_count: *mut u32, soft_count: *mut u32) -> c_int;
    pub fn ks_node_bind(s: *mut ks_snapshot, pods: *const ks_pods, group: *const i32, n_groups: u32,
                        topo: *const ks_spread_multi, aff: *const ks_pod_affinity, scoring: *const ks_bind_scoring,
                        rules: *const ks_node_rules, policy: c_int, node_idx: *mut i32, score: *mut i64,
                        parts: *mut i64, refused: *mut u32, domain_count: *mut u32, soft_count: *mut u32) -> c_int;
    pub fn ks_fit_bind(s: *mut ks_snapshot, pods: *const ks_pods, group: *const i32, n_groups: u32,
                       topo: *const ks_spread_multi, aff: *const ks_pod_affinity, scoring: *const ks_bind_scoring,
                       rules: *const ks_node_rules, res: *const ks_bind_resources, policy: c_int, node_idx: *mut i32,
                       score: *mut i64, parts: *mut i64, refused: *mut u32, domain_count: *mut u32,
                       soft_count: *mut u32, free: *mut i64) -> c_int;
    // ks_fit_bind with gangs placed all or nothing (DESIGN.md 5s)
    pub fn ks_gang_fit_bind(s: *mut ks_snapshot, pods: *const ks_pods, group: *const i32, n_groups: u32,
                            topo: *const ks_spread_multi, aff: *const ks_pod_affinity, scoring: *const ks_bind_scoring,
                            rules: *const ks_node_rules, res: *const ks_bind_resources, gangs: *const ks_gangs,
                            policy: c_int, node_idx: *mut i32, score: *mut i64, parts: *mut i64, refused: *mut u32,
                            domain_count: *mut u32, soft_count: *mut u32, free: *mut i64, placed: *mut u32) -> c_int;
    // ks_preempt under the full filter: pod count, scalar resources, taints and required node affinity (DESIGN.md 5t)
    pub fn ks_fit_preempt(s: *mut ks_snapshot, pods: *const ks_pods, group: *const i32, n_groups: u32,
                          rules: *const ks_node_rules, res: *const ks_bind_resources, pod_priority: *const i32,
                          bound: *const ks_bound_pods, bound_req: *const i64, max_victims: u32,
                          out: *mut ks_preemption, out_victims: *mut i32, out_unresolvable: *mut u32) -> c_int;
    // ks_drain_check under the full filter: pod count, scalar resources, taints and required node affinity (DESIGN.md 5u)
    pub fn ks_fit_drain_check(s: *mut ks_snapshot, pods: *const ks_pods, group: *const i32, n_groups: u32,
                              rules: *const ks_node_rules, res: *const ks_bind_resources,
                              cand: *const ks_drain_candidates, policy: c_int, flags: u32, out_placed: *mut u32,
                              out_node_idx: *mut i32, out_score: *mut i64, out_refused: *mut u32) -> c_int;
    // ks_scaleup_estimate under the full filter, with the templates as the nodes of rules and res (DESIGN.md 5v)
    pub fn ks_fit_scaleup_estimate(s: *mut ks_snapshot, pods: *const ks_pods, group: *const i32, n_groups: u32,
                                   rules: *const ks_node_rules, res: *const ks_bind_resources,
                                   t: *const ks_node_templates, out: *mut ks_scaleup_option, best: *mut i32,
                                   node: *mut i32, out_refused: *mut u32, out_used: *mut i64) -> c_int;
    // asynchronous streaming surface = the Controller's work queue (src/main.rs:73,141-148)
    pub fn ks_stream_open(s: *mut ks_snapshot, policy: c_int, max_batch: u32, out: *mut *mut ks_stream) -> c_int;
    pub fn ks_stream_submit(q: *mut ks_stream, n: u64, cpu: *const i64, mem: *const i64, sel: *const u64, tickets: *const u64) -> c_int;
    pub fn ks_stream_poll(q: *mut ks_stream, max: u64, ticket: *mut u64, node_idx: *mut i32, score: *mut i64, out_n: *mut u64) -> c_int;
    pub fn ks_stream_flush(q: *mut ks_stream) -> c_int;
    pub fn ks_stream_close(q: *mut ks_stream);
    // multi-GPU: CUDA-IPC gather buffers for ks_bindings.exchange
    pub fn ks_ipc_alloc(device: c_int, bytes: u64, out_ptr: *mut *mut c_void, out_handle: *mut u8) -> c_int;
    pub fn ks_ipc_open(device: c_int, handle: *const u8, out_ptr: *mut *mut c_void) -> c_int;
    pub fn ks_ipc_close(device: c_int, ptr: *mut c_void) -> c_int;
    pub fn ks_ipc_free(device: c_int, ptr: *mut c_void) -> c_int;
    pub fn ks_exchange_check(s: *mut ks_snapshot) -> c_int;
    // ---- object layer (include/ksched_host.h) ----
    pub fn ksh_context_create(device: c_int, out: *mut *mut ksh_context) -> c_int;
    pub fn ksh_context_destroy(ctx: *mut ksh_context);
    pub fn ksh_context_set_nodes(ctx: *mut ksh_context, nodes: *const ks_node_obj, n: u32) -> c_int;
    pub fn ksh_context_set_cluster_pods(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64) -> c_int;
    pub fn ksh_context_upsert_node(ctx: *mut ksh_context, node: *const ks_node_obj, out_idx: *mut u32) -> c_int;
    pub fn ksh_context_remove_node(ctx: *mut ksh_context, name: *const c_char) -> c_int;
    pub fn ksh_context_pod_bound(ctx: *mut ksh_context, pod: *const ks_pod_obj) -> c_int;
    pub fn ksh_context_pod_deleted(ctx: *mut ksh_context, pod: *const ks_pod_obj) -> c_int;
    pub fn ksh_context_node_name(ctx: *const ksh_context, node_idx: u32) -> *const c_char;
    pub fn ksh_context_num_nodes(ctx: *const ksh_context) -> u32;
    pub fn ksh_total_pod_resources(pod: *const ks_pod_obj, cpu: *mut i64, mem: *mut i64) -> c_int;
    pub fn ksh_is_pod_bound(pod: *const ks_pod_obj) -> c_int;
    pub fn ksh_check_node_validity(ctx: *mut ksh_context, pod: *const ks_pod_obj, node_idx: u32) -> c_int;
    pub fn ksh_select_nodes(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, policy: c_int,
                            node_idx: *mut i32, score: *mut i64, cnt: *mut u32) -> c_int;
    pub fn ksh_rank_nodes(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, policy: c_int, k: u32,
                          node_idx: *mut i32, score: *mut i64, cnt: *mut u32) -> c_int;
    pub fn ksh_context_set_pod_priorities(ctx: *mut ksh_context, pods: *const ks_pod_obj, priority: *const i32, n: u64) -> c_int;
    pub fn ksh_preempt_pods(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, pod_priority: *const i32, max_victims: u32,
                            out: *mut ks_preemption, victims: *mut c_char, cap: usize, out_victim_off: *mut i64) -> c_int;
    pub fn ksh_select_node_for_pod(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, attempts: u32, seed: u64,
                                   first_pod_index: u64, node_idx: *mut i32, attempts_used: *mut u32,
                                   draw_node: *mut i32, draw_code: *mut u8) -> c_int;
    pub fn ksh_reconcile(ctx: *mut ksh_context, pod: *const ks_pod_obj, policy: c_int, node_idx: *mut i32,
                         binding_json: *mut c_char, cap: usize) -> c_int;
    pub fn ksh_reconcile_batch(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, policy: c_int, status: *mut i32,
                               node_idx: *mut i32, json: *mut c_char, cap: usize, json_off: *mut i64, rounds: *mut u32) -> c_int;
    pub fn ksh_reconcile_gangs(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, group_offset: *const u64, n_groups: u64,
                               min_member: *const u32, policy: c_int, status: *mut i32, node_idx: *mut i32, placed: *mut u32,
                               json: *mut c_char, cap: usize, json_off: *mut i64) -> c_int;
    pub fn ksh_context_snapshot(ctx: *mut ksh_context) -> *mut ks_snapshot; // borrowed, until the next mutation
    pub fn ksh_scaleup_estimate(ctx: *mut ksh_context, templates: *const ks_node_obj, n_templates: u64, max_nodes: *const u32,
                                overhead_pods: *const ks_pod_obj, n_overhead: u64, pods: *const ks_pod_obj, n_pods: u64,
                                out: *mut ks_scaleup_option, best: *mut i32, node: *mut i32,
                                reasons: *mut ks_pod_reasons) -> c_int;
    pub fn ksh_place_replicas(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, replicas: *const u32, policy: c_int,
                              out: *mut ks_replica_plan, node: *mut i32, score: *mut i64) -> c_int;
    pub fn ksh_context_topology_domains(ctx: *const ksh_context, key: *const c_char, node_domain: *mut i32,
                                        n_domains: *mut u32, names: *mut c_char, cap: usize, name_off: *mut i64) -> c_int;
    pub fn ksh_place_replicas_spread(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, replicas: *const u32,
                                     topology_key: *const c_char, max_skew: *const u32, min_domains: *const u32,
                                     existing_node_names: *const *const c_char, existing_offset: *const u64, policy: c_int,
                                     out: *mut ks_spread_plan, node: *mut i32, score: *mut i64,
                                     domain_count: *mut u32) -> c_int;
    pub fn ksh_place_replicas_spread_multi(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, replicas: *const u32,
                                           topology_keys: *const *const c_char, n_keys: u32, max_skew: *const u32,
                                           min_domains: *const u32, existing_node_names: *const *const c_char,
                                           existing_offset: *const u64, policy: c_int, out: *mut ks_spread_plan,
                                           node: *mut i32, score: *mut i64, domain_count: *mut u32) -> c_int;
    pub fn ksh_reconcile_spread(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, group: *const i32, n_groups: u32,
                                topology_keys: *const *const c_char, n_keys: u32, max_skew: *const u32,
                                min_domains: *const u32, existing_node_names: *const *const c_char,
                                existing_offset: *const u64, policy: c_int, status: *mut i32, node_idx: *mut i32,
                                json: *mut c_char, cap: usize, json_off: *mut i64) -> c_int;
    pub fn ksh_reconcile_affinity(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, group: *const i32,
                                  n_groups: u32, topology_keys: *const *const c_char, n_keys: u32, max_skew: *const u32,
                                  min_domains: *const u32, existing_node_names: *const *const c_char,
                                  existing_offset: *const u64, aff: *const ksh_pod_affinity, policy: c_int,
                                  status: *mut i32, node_idx: *mut i32, json: *mut c_char, cap: usize,
                                  json_off: *mut i64) -> c_int;
    pub fn ksh_context_set_node_taints(ctx: *mut ksh_context, node_names: *const *const c_char, taint_offset: *const u64,
                                       taints: *const ksh_taint, n: u64) -> c_int;
    pub fn ksh_compile_node_rules(ctx: *mut ksh_context, n_groups: u32, rules: *const ksh_node_rules, hard: *mut u8,
                                  affinity: *mut u8, soft: *mut u32, preferred: *mut u32) -> c_int;
    pub fn ksh_reconcile_nodes(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, group: *const i32, n_groups: u32,
                               topology_keys: *const *const c_char, n_keys: u32, max_skew: *const u32,
                               min_domains: *const u32, existing_node_names: *const *const c_char,
                               existing_offset: *const u64, aff: *const ksh_pod_affinity,
                               scoring: *const ks_bind_scoring, rules: *const ksh_node_rules, policy: c_int,
                               status: *mut i32, node_idx: *mut i32, json: *mut c_char, cap: usize,
                               json_off: *mut i64) -> c_int;
    pub fn ksh_compile_resources(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, names: *mut c_char, cap: usize,
                                 node_free: *mut i64, pod_req: *mut i64) -> c_int;
    pub fn ksh_reconcile_fit(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, group: *const i32, n_groups: u32,
                             topology_keys: *const *const c_char, n_keys: u32, max_skew: *const u32,
                             min_domains: *const u32, existing_node_names: *const *const c_char,
                             existing_offset: *const u64, aff: *const ksh_pod_affinity,
                             scoring: *const ks_bind_scoring, rules: *const ksh_node_rules, policy: c_int,
                             status: *mut i32, node_idx: *mut i32, json: *mut c_char, cap: usize,
                             json_off: *mut i64) -> c_int;
    pub fn ksh_reconcile_fit_gangs(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, group: *const i32,
                                   n_groups: u32, topology_keys: *const *const c_char, n_keys: u32,
                                   max_skew: *const u32, min_domains: *const u32,
                                   existing_node_names: *const *const c_char, existing_offset: *const u64,
                                   aff: *const ksh_pod_affinity, scoring: *const ks_bind_scoring,
                                   rules: *const ksh_node_rules, gang_offset: *const u64, n_gangs: u64,
                                   min_member: *const u32, policy: c_int, status: *mut i32, node_idx: *mut i32,
                                   placed: *mut u32, json: *mut c_char, cap: usize, json_off: *mut i64) -> c_int;
    // ksh_preempt_pods under the full filter: taints, node affinity, extended resources and the pod limit (DESIGN.md 5t)
    pub fn ksh_preempt_fit_pods(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, group: *const i32,
                                n_groups: u32, rules: *const ksh_node_rules, pod_priority: *const i32,
                                max_victims: u32, out: *mut ks_preemption, victims: *mut c_char, cap: usize,
                                out_victim_off: *mut i64) -> c_int;
    pub fn ksh_reconcile_profile(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, group: *const i32,
                                 n_groups: u32, topology_keys: *const *const c_char, n_keys: u32, max_skew: *const u32,
                                 min_domains: *const u32, existing_node_names: *const *const c_char,
                                 existing_offset: *const u64, aff: *const ksh_pod_affinity,
                                 scoring: *const ks_bind_scoring, policy: c_int, status: *mut i32, node_idx: *mut i32,
                                 json: *mut c_char, cap: usize, json_off: *mut i64) -> c_int;
    pub fn ksh_drain_nodes(ctx: *mut ksh_context, node_names: *const *const c_char, n: u64, pods: *const ks_pod_obj,
                           pod_offset: *const u64, policy: c_int, flags: u32, placed: *mut u32, node_idx: *mut i32) -> c_int;
    // ksh_drain_nodes under the full filter: taints, node affinity, extended resources and the pod limit (DESIGN.md 5u)
    pub fn ksh_drain_fit_nodes(ctx: *mut ksh_context, node_names: *const *const c_char, n: u64, pods: *const ks_pod_obj,
                               pod_offset: *const u64, group: *const i32, n_groups: u32, rules: *const ksh_node_rules,
                               policy: c_int, flags: u32, placed: *mut u32, node_idx: *mut i32,
                               refused: *mut u32) -> c_int;
    pub fn ksh_scaleup_fit_estimate(ctx: *mut ksh_context, templates: *const ks_node_obj, n_templates: u64,
                                    max_nodes: *const u32, template_taint_offset: *const u64,
                                    template_taints: *const ksh_taint, overhead_pods: *const ks_pod_obj,
                                    n_overhead: u64, pods: *const ks_pod_obj, n_pods: u64, group: *const i32,
                                    n_groups: u32, rules: *const ksh_node_rules, out: *mut ks_scaleup_option,
                                    best: *mut i32, node: *mut i32, refused: *mut u32) -> c_int;
    pub fn ksh_explain_pods(ctx: *mut ksh_context, pods: *const ks_pod_obj, n: u64, out: *mut ks_pod_reasons,
                            messages: *mut c_char, cap: usize, msg_off: *mut i64) -> c_int;
    pub fn ksh_format_unschedulable(n_nodes: u32, r: *const ks_pod_reasons, buf: *mut c_char, cap: usize) -> c_int;
}
