/* ksched_host.h — host layer of libksched.so: the reference's scheduling surface over Pod/Node OBJECTS.
 *
 * The reference's host is Rust (async fns inside a binary crate).  No Rust toolchain exists in this image,
 * so this layer is C++ behind a C ABI that keeps the reference's names, argument meaning and error
 * behaviour; a Rust controller would bind it with the `extern "C"` block shown in INTEGRATION.md and keep
 * its reconcile() loop.  Mapping (paths relative to /root/reference):
 *   ksh_total_pod_resources   <- total_pod_resources            src/util.rs:54-75
 *   ksh_is_pod_bound          <- is_pod_bound                   src/util.rs:38-45
 *   ksh_context               <- Context{client,node_store}     src/util.rs:12-15 (+ the LIST of src/predicates.rs:21-38)
 *   ksh_check_node_validity   <- check_node_validity            src/predicates.rs:63-77
 *   ksh_select_nodes          <- select_node_for_pod, batched   src/main.rs:51-71 (argmax score instead of 5 random draws)
 *   ksh_select_node_for_pod   <- select_node_for_pod, seeded    src/main.rs:49-71 (the reference's own 5-draw policy)
 *   ksh_reconcile_batch       <- reconcile over a drained queue  src/main.rs:73-120 (micro-batch with capacity commit)
 *   ksh_reconcile             <- reconcile                      src/main.rs:73-120 (builds the Binding, does not POST it)
 *   KSH_RECONCILE_*           <- ReconcileError                 src/error.rs:5-15
 * The layer packs objects into the SoA/bitmask form of ksched.h and calls the CUDA core; it never evaluates
 * a predicate on the CPU.  Malformed quantities / missing allocatable keys (reference: panic) return
 * KS_ERR_PARSE / KS_ERR_MISSING at pack time.
 */
#ifndef KSCHED_HOST_H
#define KSCHED_HOST_H

#include <stddef.h>
#include <stdint.h>

#include "ks_objects.h"
#include "ksched.h"

#ifdef __cplusplus
extern "C" {
#endif

/* reconcile outcomes: Ok(Action::await_change()) or ReconcileError (src/error.rs:5-15) */
#define KSH_RECONCILE_OK 0                   /* pod already bound (src/main.rs:74-76) or binding produced */
#define KSH_RECONCILE_NO_NODE_FOUND 1        /* ReconcileError::NoNodeFound (src/main.rs:116-118) */
#define KSH_RECONCILE_BINDING_OBJECT_FAILED 2 /* ReconcileError::CreateBindingObjectFailed (src/main.rs:111-114);
                                                 also a pod without namespace (reference: unwrap panic, :80) */
#define KSH_RECONCILE_BINDING_FAILED 3       /* ReconcileError::CreateBindingFailed: transport, caller side (:105-108) */
#define KSH_RECONCILE_GANG_UNSATISFIED 4     /* ksh_reconcile_gangs: the pod's group could not place min_member pods */
#define KSH_RECONCILE_SPREAD_UNSATISFIED 5   /* ksh_reconcile_spread: a node would take the pod but its spread constraints
                                                refused every such node (upstream: "didn't match pod topology spread
                                                constraints") */
#define KSH_RECONCILE_AFFINITY_UNSATISFIED 6 /* ksh_reconcile_affinity: fit, selector and spread passed on some node but
                                                the pod's inter-pod (anti-)affinity refused every such node (upstream:
                                                "didn't match pod affinity/anti-affinity rules") */
#define KSH_RECONCILE_NODE_RULES_UNSATISFIED 7 /* ksh_reconcile_nodes: some node fit (resources and selector) but taints
                                                  or required node affinity refused every such node (upstream:
                                                  "untolerated taint" / "didn't match Pod's node affinity/selector") */
#define KSH_RECONCILE_INSUFFICIENT_RESOURCES 8 /* ksh_reconcile_fit: some node passed cpu, memory and selector but every
                                                  such node lacked a scalar resource the pod requests or was at its pod
                                                  limit (upstream: "Insufficient nvidia.com/gpu" / "Too many pods") */

/* Kubernetes quantity strings, exact: cpu -> millicores, memory -> bytes.
 * KS_ERR_PARSE (malformed), KS_ERR_INEXACT (finer than 1m / 1 byte), KS_ERR_RANGE. */
int ksh_parse_cpu_millicores(const char* quantity, int64_t* out);
int ksh_parse_memory_bytes(const char* quantity, int64_t* out);

int ksh_total_pod_resources(const ks_pod_obj* pod, int64_t* cpu_millicores, int64_t* mem_bytes);
int ksh_is_pod_bound(const ks_pod_obj* pod);

typedef struct ksh_context ksh_context;
/* device = CUDA ordinal, or KSH_DEVICE_NONE for a packing-only context: objects -> SoA/bitmask arrays
 * (ksh_context_set_* / upsert / pod events, ksh_pack_pods, ksh_context_export_packed) work on the host; every call
 * that evaluates a predicate or selects a node returns KS_ERR_NO_DEVICE — nothing is ever computed on the CPU. */
#define KSH_DEVICE_NONE (-1)
int ksh_context_create(int device, ksh_context** out);
void ksh_context_destroy(ksh_context* ctx);
/* node store contents (what reflector::Store<Node>::state() returns, src/main.rs:56).  The store is keyed by name, so
 * names are unique; if a name repeats anyway, pods and events address the first node of that name. */
int ksh_context_set_nodes(ksh_context* ctx, const ks_node_obj* nodes, uint32_t n_nodes);
/* every pod object the API server holds; those with spec.nodeName naming a known node are the LIST results
 * of src/predicates.rs:22-34 (any phase) and are charged to that node; the rest are ignored here. */
int ksh_context_set_cluster_pods(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods);
/* Incremental node-store / informer events (what the reflector applies between reconciles, src/main.rs:133-139):
 * - upsert: add a node or replace the one with the same metadata.name; *out_idx = its index
 * - remove: delete by name; later nodes move down by one index (indices are positions in the current store;
 *   ksh_context_node_name maps an index back to the name a Binding needs)
 * - pod_bound / pod_deleted: a pod with spec.nodeName appeared / went away; capacity is charged / returned.
 *   Pods are identified by namespace/name; unknown pods or nodes are ignored (KS_OK), like a LIST that no
 *   longer shows them.
 * The device snapshot is refreshed lazily on the next select/check call. */
int ksh_context_upsert_node(ksh_context* ctx, const ks_node_obj* node, uint32_t* out_idx);
int ksh_context_remove_node(ksh_context* ctx, const char* name);
int ksh_context_pod_bound(ksh_context* ctx, const ks_pod_obj* pod);
int ksh_context_pod_deleted(ksh_context* ctx, const ks_pod_obj* pod);
const char* ksh_context_node_name(const ksh_context* ctx, uint32_t node_idx); /* NULL if out of range; borrowed,
                                                                                 valid until the next ksh_context_* mutation */
uint32_t ksh_context_num_nodes(const ksh_context* ctx);
uint32_t ksh_context_label_words(const ksh_context* ctx);
uint64_t ksh_context_num_bound(const ksh_context* ctx);
/* The packed node side exactly as the next device upload sends it (arguments of ks_snapshot_set_nodes /
 * ks_snapshot_set_bound in ksched.h): allocatable [N] in millicores / bytes, label words [N * label_words] under the
 * current dictionary, bound-pod triples [num_bound].  Lets a host feed the packed core itself, and the CPU tests
 * check the packer against the oracle without a GPU. */
int ksh_context_export_packed(const ksh_context* ctx, int64_t* alloc_cpu, int64_t* alloc_mem, uint64_t* labels,
                              int32_t* bound_node, int64_t* bound_cpu, int64_t* bound_mem);
ks_snapshot* ksh_context_snapshot(ksh_context* ctx); /* borrowed; valid until the next ksh_context_* mutation */

/* Pack P pod objects into caller buffers (req_cpu[P], req_mem[P], sel[P*W]) with the context's current label
 * dictionary, growing the dictionary (and re-uploading node columns) when a selector names a new pair.
 * Returns W (>0) on success so the caller can size `sel` = P * 8 words up front (KS_MAX_LABEL_WORDS). */
int ksh_pack_pods(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, int64_t* req_cpu, int64_t* req_mem,
                  uint64_t* sel, uint32_t sel_stride_words);

int ksh_check_node_validity(ksh_context* ctx, const ks_pod_obj* pod, uint32_t node_idx);
/* select_node_for_pod for a whole batch (src/main.rs:51-71 with the argmax over ALL feasible nodes instead of <= 5 draws):
 * out_node_idx[p] < 0 = None.  A pod whose quantities do not parse fails the call before anything is evaluated (status +
 * ks_last_error(), the reference panics there: src/util.rs:65,68).  The context keeps the packed form of the last batch
 * (24 + 8W bytes per pod) until it is destroyed, so that repeated calls do not fault in fresh pages. */
int ksh_select_nodes(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, int policy, int32_t* out_node_idx,
                     int64_t* out_score, uint32_t* out_feasible_cnt);
/* Ranked alternatives: ks_select_topk (ksched.h) over pod objects, packed as ksh_select_nodes packs them.  Row p of
 * out_node_idx[n_pods*k] lists pod p's k best feasible nodes (-1 past the feasible count), entry 0 being what
 * ksh_select_nodes picks; map indices to names with ksh_context_node_name.  Nothing is charged: after a Binding POST
 * for one of them succeeds, report it with ksh_context_pod_bound.  out_score[n_pods*k] / out_feasible_cnt[n_pods] may
 * be NULL.  KS_ERR_NO_DEVICE on a packing-only context. */
int ksh_rank_nodes(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, int policy, uint32_t k,
                   int32_t* out_node_idx, int64_t* out_score, uint32_t* out_feasible_cnt);

/* select_node_for_pod with the reference's OWN policy (src/main.rs:49-71): <= attempts seeded random draws per pod,
 * first valid draw wins, -1 = None.  Arguments as ks_select_sampling (ksched.h); pass KS_REFERENCE_ATTEMPTS for the
 * reference's ATTEMPTS.  out_draw_code holds the InvalidNodeReason of each failed draw (what src/main.rs:62 logs). */
int ksh_select_node_for_pod(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, uint32_t attempts, uint64_t seed,
                            uint64_t first_pod_index, int32_t* out_node_idx, uint32_t* out_attempts,
                            int32_t* out_draw_node, uint8_t* out_draw_code);

/* One reconcile: skip bound pods, select, emit `POST /api/v1/namespaces/{ns}/pods/{name}/binding` body, and
 * charge the pod to the chosen node in the snapshot (what the next LIST would show).  *node_idx = -1 if none.
 * binding_json may be NULL; otherwise receives a NUL-terminated JSON document (truncated to cap). */
int ksh_reconcile(ksh_context* ctx, const ks_pod_obj* pod, int policy, int32_t* node_idx, char* binding_json,
                  size_t cap);

/* reconcile() for a drained controller queue, pods in arrival order.  Pods already bound are skipped (KSH_RECONCILE_OK,
 * node -1; src/main.rs:74-76); pods without namespace/name get KSH_RECONCILE_BINDING_OBJECT_FAILED (reference: unwrap
 * panic, :80) and are not scheduled; the rest are packed once and bound by the micro-batch loop of ks_stream_bind (ksched.h):
 * every round selects on the current capacity, claims are accepted per node in arrival order while they still fit, losers
 * are re-selected against what is left — capacity is never oversubscribed, a pod ends with KSH_RECONCILE_NO_NODE_FOUND
 * only if no node fits it at its turn.  Accepted binds are committed to the snapshot and to the context's bound-pod list.
 * out_status[n], out_node_idx[n] (-1 = none).  Binding bodies (see ksh_reconcile) are written back to back, NUL-terminated,
 * into json (cap bytes); out_json_off[i] = offset of pod i's body or -1 (not bound, or the buffer was full).  json /
 * out_json_off / out_rounds may be NULL. */
int ksh_reconcile_batch(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, int policy, int32_t* out_status,
                        int32_t* out_node_idx, char* json, size_t cap, int64_t* out_json_off, uint32_t* out_rounds);

/* reconcile() for pod groups, all or nothing (ks_gang_bind, ksched.h; upstream coscheduling's PodGroup minMember).  Group
 * g is pods [group_offset[g], group_offset[g+1]), 1..KS_GANG_MAX_SIZE of them, min_member[g] <= its size; groups run in
 * order.  Pods are filtered as ksh_reconcile_batch filters them: already bound pods are skipped (KSH_RECONCILE_OK, node
 * -1) but count toward their group's min_member, as running members do upstream; pods without namespace/name get
 * KSH_RECONCILE_BINDING_OBJECT_FAILED and do not count.  The rest of each group goes to the device with
 * max(0, min_member - bound members).  A group that commits binds as ksh_reconcile_batch does (charged to the snapshot
 * and the bound list at priority 0, Binding bodies in json / out_json_off, KSH_RECONCILE_NO_NODE_FOUND for its unplaced
 * pods); a group that rolls back - or has fewer schedulable members than it still needs - binds nothing, and those
 * pods get KSH_RECONCILE_GANG_UNSATISFIED.  As in ksh_reconcile_batch, every unbound pod with a namespace and name first
 * loses any charge this context made earlier for it (it came back unbound), whatever its group's outcome.  out_placed[n_groups] (may be NULL) = pods the device placed before any
 * rollback.  Offsets and sizes are checked first: KS_ERR_INVALID (offsets) / KS_ERR_RANGE (sizes, min_member);
 * KS_ERR_NO_DEVICE on a packing-only context. */
int ksh_reconcile_gangs(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, const uint64_t* group_offset,
                        uint64_t n_groups, const uint32_t* min_member, int policy, int32_t* out_status,
                        int32_t* out_node_idx, uint32_t* out_placed, char* json, size_t cap, int64_t* out_json_off);

/* Why pods do not schedule: ks_explain (ksched.h) over pod objects, packed as ksh_select_nodes packs them (a selector
 * pair that no node carries counts as a selector mismatch on every node).  out[n_pods] receives the counts.  For each
 * pod with no feasible node, a FailedScheduling message (ksh_format_unschedulable) is written into messages (cap bytes),
 * back to back and NUL-terminated like ksh_reconcile_batch's bodies; out_msg_off[i] = its offset, or -1 (the pod has a
 * feasible node, or the buffer was full).  messages / out_msg_off may be NULL. */
int ksh_explain_pods(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, ks_pod_reasons* out, char* messages,
                     size_t cap, int64_t* out_msg_off);
/* Upstream kube-scheduler's message for a pod no node accepts, e.g.
 *   "0/5 nodes are available: 2 Insufficient cpu, 3 node(s) didn't match Pod's node affinity/selector."
 * "0/<n_nodes> nodes are available: " then the non-zero terms of insufficient_cpu ("<a> Insufficient cpu"),
 * insufficient_memory ("<b> Insufficient memory") and node_selector_mismatch ("<c> node(s) didn't match Pod's node
 * affinity/selector"), joined by ", ", ended by "."; with no term (n_nodes = 0) "0/<n_nodes> nodes are available.".
 * Pure CPU.  Like snprintf: writes at most cap bytes including the NUL and returns the full length (>= cap means
 * truncated); KS_ERR_INVALID when r is NULL, or buf is NULL with cap > 0. */
int ksh_format_unschedulable(uint32_t n_nodes, const ks_pod_reasons* r, char* buf, size_t cap);

/* Priority preemption over pod objects (ks_preempt, ksched.h).
 * ksh_context_set_pod_priorities records spec.priority for bound pods known by namespace/name; unknown pods are ignored
 * (KS_OK), as with the other events.  A bound pod's priority is 0 until it is set, follows its pod through pod events
 * (a repeated ksh_context_pod_bound for the same pod keeps it: spec.priority is immutable), and is reset to 0 by
 * ksh_context_set_nodes / ksh_context_set_cluster_pods, which rebuild the bound list, and for pods that
 * ksh_reconcile / ksh_reconcile_batch bind.  Bound pods without namespace and name cannot be named for eviction, so they
 * are passed as priority INT32_MAX and are never victims.
 * ksh_preempt_pods packs pods as ksh_select_nodes does and passes the context's bound pods as the ks_bound_pods list;
 * pod_priority[n_pods] is each pending pod's priority.  out[n_pods] receives the plans (node index: map it with
 * ksh_context_node_name).  For each pod with a plan, its victims' "namespace/name" keys are written into victims (cap
 * bytes) back to back, each NUL-terminated, in visit order; out_victim_off[i] = offset of pod i's first key, or -1 (no
 * plan, or the buffer was full).  victims / out_victim_off may be NULL.  Nothing is charged: DELETE the victims, report
 * each with ksh_context_pod_deleted, and requeue the pod.  KS_ERR_RANGE for max_victims outside
 * [1, KS_PREEMPT_MAX_VICTIMS]; KS_ERR_NO_DEVICE on a packing-only context. */
int ksh_context_set_pod_priorities(ksh_context* ctx, const ks_pod_obj* pods, const int32_t* priority, uint64_t n_pods);
int ksh_preempt_pods(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, const int32_t* pod_priority,
                     uint32_t max_victims, ks_preemption* out, char* victims, size_t cap, int64_t* out_victim_off);

/* Node drain and scale-down checks over objects (ks_drain_check, ksched.h): candidate d is the node named node_names[d]
 * and owns pods [pod_offset[d], pod_offset[d+1]) (normally the pods bound to it, already filtered by the caller for
 * PodDisruptionBudgets, DaemonSet and mirror pods, local storage), packed as ksh_select_nodes packs them.  Every pod
 * must have spec.nodeName equal to its candidate's name and every name must be in the store; either failure is
 * KS_ERR_INVALID before anything else, and ks_last_error() names the offender.  out_placed[n] and out_node_idx[
 * pod_offset[n]] as ks_drain_check gives them (destinations map to names with ksh_context_node_name); candidate d is
 * drainable iff out_placed[d] is its pod count.  Nothing is charged.  KS_ERR_NO_DEVICE on a packing-only context. */
int ksh_drain_nodes(ksh_context* ctx, const char* const* node_names, uint64_t n, const ks_pod_obj* pods,
                    const uint64_t* pod_offset, int policy, uint32_t flags, uint32_t* out_placed, int32_t* out_node_idx);

/* Node-group scale-up estimate over objects (ks_scaleup_estimate, ksched.h): template t is the Node object templates[t]
 * (one new node of a group; its labels are those a new node would carry, instance type included) with max_nodes[t].
 * Allocatable is parsed as ksh_context_set_nodes parses it (a missing cpu or memory key is KS_ERR_MISSING; a template
 * without allocatable has allocatable 0, which ks_scaleup_estimate refuses with KS_ERR_RANGE).  Each overhead pod (a
 * DaemonSet pod) has spec.nodeName equal to a template's name and its total_pod_resources is charged to that template,
 * so capacity = allocatable - the sum, as upstream builds a template's NodeInfo.  The pending pods are packed against a
 * call-local dictionary: one bit per (key, value) pair that some pending pod's selector names and some template
 * carries, in the order the pods name them; every other selector pair maps to the never-set bit (more than 511 such
 * pairs is KS_ERR_RANGE).  KS_ERR_INVALID before any device work for a NULL argument or name, duplicate template
 * names, an overhead pod without spec.nodeName or naming an unknown template, or a pending pod with spec.nodeName set;
 * ks_last_error() names the offender.  A malformed quantity fails with its parse status first as well.  The context's
 * node store, dictionary, bound list and snapshot are not changed.  Outputs as ks_scaleup_estimate gives them
 * (out[n_templates] required when n_templates > 0, out_best required, out_node[n_templates * n_pods] and
 * out_reasons[n_pods] may be NULL).  KS_ERR_NO_DEVICE on a packing-only context. */
int ksh_scaleup_estimate(ksh_context* ctx, const ks_node_obj* templates, uint64_t n_templates, const uint32_t* max_nodes,
                         const ks_pod_obj* overhead_pods, uint64_t n_overhead, const ks_pod_obj* pods, uint64_t n_pods,
                         ks_scaleup_option* out, int32_t* out_best, int32_t* out_node, ks_pod_reasons* out_reasons);

/* Replica placement over objects (ks_place_replicas, ksched.h): spec t is pods[t] with replicas[t] copies, packed as
 * ksh_select_nodes packs them (a selector pair no node carries maps to the never-set bit, so that spec's capacity is 0).
 * Nothing is charged: the bound list, the store and free[] are unchanged.  Outputs as ks_place_replicas gives them
 * (out[n] required when n > 0; out_node and out_score [sum of replicas] may be NULL; node indices map to names with
 * ksh_context_node_name).  KS_ERR_NO_DEVICE on a packing-only context. */
int ksh_place_replicas(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n, const uint32_t* replicas, int policy,
                       ks_replica_plan* out, int32_t* out_node, int64_t* out_score);

/* The domains of one topology key (e.g. "topology.kubernetes.io/zone", "kubernetes.io/hostname") over the node store:
 * nodes whose labels carry `key' get dense ids 0..D-1, numbered by the value's first appearance in node-index order;
 * every other node gets -1.  out_node_domain[N] (N = ksh_context_num_nodes) and *out_n_domains receive them.  The
 * values are written into names (cap bytes) back to back, NUL-terminated like ksh_reconcile_batch's bodies;
 * out_name_off[d] = offset of domain d's value, or -1 (the buffer was full); D <= N, so N entries always suffice.
 * names / out_name_off may be NULL.  Pure host work: works on a packing-only context.  Node upserts and removals
 * renumber the domains of later calls. */
int ksh_context_topology_domains(const ksh_context* ctx, const char* key, int32_t* out_node_domain,
                                 uint32_t* out_n_domains, char* names, size_t cap, int64_t* out_name_off);

/* Replica placement under one topology spread constraint over objects (ks_place_replicas_spread, ksched.h): spec t is
 * pods[t] with replicas[t] copies, packed as ksh_place_replicas packs them, spread over the domains of topology_key as
 * ksh_context_topology_domains numbers them, with max_skew[t] and min_domains[t] (min_domains may be NULL).  The nodes
 * of the bound pods that match spec t's constraint selector are existing_node_names[existing_offset[t] ..
 * existing_offset[t+1]) (ks_pod_obj carries no pod labels, so the caller filters the pods); a name not in the store,
 * or a node without the key, is not counted.  existing_offset [n + 1] may be NULL (no existing pods).  Nothing is
 * charged.  Outputs as ks_place_replicas_spread gives them (out[n] required when n > 0; out_node, out_score [sum of
 * replicas] and out_domain_count [n * D] may be NULL).  With no node carrying the key, every row is empty and
 * out_domain_count is not written.  KS_ERR_NO_DEVICE on a packing-only context. */
int ksh_place_replicas_spread(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n, const uint32_t* replicas,
                              const char* topology_key, const uint32_t* max_skew, const uint32_t* min_domains,
                              const char* const* existing_node_names, const uint64_t* existing_offset, int policy,
                              ks_spread_plan* out, int32_t* out_node, int64_t* out_score, uint32_t* out_domain_count);

/* The same over n_keys topology keys at once (ks_place_replicas_spread_multi, ksched.h), such as
 * topology.kubernetes.io/zone and kubernetes.io/hostname: key k is topology_keys[k], numbered as
 * ksh_context_topology_domains numbers it; max_skew [n * K] and min_domains [n * K] (or NULL) per (spec, key).  Spec t's
 * existing pods under key k are existing_node_names[existing_offset[t * K + k] .. existing_offset[t * K + k + 1])
 * (existing_offset [n * K + 1] or NULL); a name counts when it is in the store and its node carries every key of the
 * call.  Outputs as ks_place_replicas_spread_multi gives them (out [n * K], out_domain_count [n * S]).  With a key that
 * no node carries, every row is empty and out_domain_count is not written.  K = 1 gives exactly what
 * ksh_place_replicas_spread gives.  KS_ERR_RANGE for n_keys outside [1, KS_SPREAD_MAX_KEYS]; KS_ERR_NO_DEVICE on a
 * packing-only context. */
int ksh_place_replicas_spread_multi(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n, const uint32_t* replicas,
                                    const char* const* topology_keys, uint32_t n_keys, const uint32_t* max_skew,
                                    const uint32_t* min_domains, const char* const* existing_node_names,
                                    const uint64_t* existing_offset, int policy, ks_spread_plan* out, int32_t* out_node,
                                    int64_t* out_score, uint32_t* out_domain_count);

/* reconcile() under topology spread (ks_spread_bind, ksched.h): ksh_reconcile_batch with each workload's spread
 * constraints.  Pod i belongs to group group[i] in [-1, n_groups) (-1 = no constraint; KS_ERR_INVALID otherwise), and
 * every pod of a group must carry the same node selector.  Key k is topology_keys[k], numbered as
 * ksh_context_topology_domains numbers it; max_skew [n_groups * K] (0 = the group does not constrain that key) and
 * min_domains [n_groups * K] (or NULL) per (group, key).  Group g's existing pods under key k are
 * existing_node_names[existing_offset[g * K + k] .. existing_offset[g * K + k + 1]) (existing_offset [n_groups * K + 1] or
 * NULL; ks_pod_obj carries no pod labels, so the caller filters the pods); a name counts when it is in the store and its
 * node carries key k and every key the group constrains.  Pods are filtered as ksh_reconcile_batch filters them: already
 * bound pods are skipped (KSH_RECONCILE_OK, node -1) and count only when the caller lists them in existing; pods without
 * namespace/name get KSH_RECONCILE_BINDING_OBJECT_FAILED.  The rest are bound one at a time in arrival order on the
 * device, each against the capacity and counts every earlier pod left; binds are charged to the snapshot and the bound
 * list, with Binding bodies in json / out_json_off, as ksh_reconcile_batch does.  An unbound pod gets
 * KSH_RECONCILE_SPREAD_UNSATISFIED when some node passed fit and selector but its constraints refused every such node,
 * else KSH_RECONCILE_NO_NODE_FOUND.  KS_ERR_RANGE for n_keys outside [1, KS_SPREAD_MAX_KEYS]; KS_ERR_NO_DEVICE on a
 * packing-only context. */
int ksh_reconcile_spread(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, const int32_t* group,
                         uint32_t n_groups, const char* const* topology_keys, uint32_t n_keys, const uint32_t* max_skew,
                         const uint32_t* min_domains, const char* const* existing_node_names,
                         const uint64_t* existing_offset, int policy, int32_t* out_status, int32_t* out_node_idx,
                         char* json, size_t cap, int64_t* out_json_off);

/* reconcile() under topology spread and required inter-pod affinity (ks_affinity_bind, ksched.h): ksh_reconcile_spread
 * with the terms of aff (or NULL: none), and max_skew may be NULL (no spread constraint).  Term t of group owner[t] is
 * kind[t] (KS_POD_AFFINITY / KS_POD_ANTI_AFFINITY) on topology_keys[key[t]] and targets the groups
 * target[target_offset[t] .. target_offset[t + 1]), resolved by the caller from the term's labelSelector and
 * namespaces.  Existing pod e is of group existing_group[e] and bound to the node named existing_node_name[e]; a name
 * not in the store is skipped.  An unbound pod gets KSH_RECONCILE_SPREAD_UNSATISFIED when its spread constraints refused
 * some node that fit it, else KSH_RECONCILE_AFFINITY_UNSATISFIED when its affinity terms refused some node that passed
 * fit, selector and spread, else KSH_RECONCILE_NO_NODE_FOUND.  Errors as ksh_reconcile_spread and ks_affinity_bind. */
typedef struct ksh_pod_affinity {
    uint32_t n_terms;
    const int32_t* owner;              /* [T] */
    const uint8_t* kind;               /* [T] */
    const uint32_t* key;               /* [T] index into topology_keys */
    const uint64_t* target_offset;     /* [T + 1] */
    const int32_t* target;
    uint64_t n_existing;               /* E */
    const int32_t* existing_group;     /* [E] */
    const char* const* existing_node_name; /* [E] */
} ksh_pod_affinity;
int ksh_reconcile_affinity(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, const int32_t* group,
                           uint32_t n_groups, const char* const* topology_keys, uint32_t n_keys,
                           const uint32_t* max_skew /* or NULL */, const uint32_t* min_domains,
                           const char* const* existing_node_names, const uint64_t* existing_offset,
                           const ksh_pod_affinity* aff, int policy, int32_t* out_status, int32_t* out_node_idx,
                           char* json, size_t cap, int64_t* out_json_off);

/* reconcile() under topology spread, required inter-pod affinity and the default profile's soft scores
 * (ks_profile_bind, ksched.h): ksh_reconcile_affinity with term kinds 0 to 3 (KS_POD_AFFINITY_PREFERRED /
 * KS_POD_ANTI_AFFINITY_PREFERRED score only) and a scoring struct (required; its term_weight is indexed as aff's terms,
 * its soft_skew and soft_all_keys by group and topology_keys).  The soft counts start from the same existing counts as
 * the hard ones.  Soft terms never make a pod unschedulable, so the status mapping is ksh_reconcile_affinity's.  Errors
 * as ksh_reconcile_affinity and ks_profile_bind; KS_ERR_INVALID for a NULL scoring. */
int ksh_reconcile_profile(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, const int32_t* group,
                          uint32_t n_groups, const char* const* topology_keys, uint32_t n_keys,
                          const uint32_t* max_skew /* or NULL */, const uint32_t* min_domains,
                          const char* const* existing_node_names, const uint64_t* existing_offset,
                          const ksh_pod_affinity* aff /* or NULL */, const ks_bind_scoring* scoring, int policy,
                          int32_t* out_status, int32_t* out_node_idx, char* json, size_t cap, int64_t* out_json_off);

/* Taints and node affinity over objects (ks_node_bind, ksched.h; DESIGN.md 5p).
 * ksh_context_set_node_taints records spec.taints of nodes in the store: node node_names[i] carries
 * taints[taint_offset[i] .. taint_offset[i + 1]), replacing what it carried.  Names not in the store are ignored (KS_OK),
 * as with the other events.  A node's taints are kept by name: they survive an upsert of that name, are dropped by
 * ksh_context_remove_node and are cleared by ksh_context_set_nodes.  A taint needs a non-empty key and the effect
 * NoSchedule, PreferNoSchedule or NoExecute (KS_ERR_INVALID otherwise, before anything changes); a NULL value is "".
 * Pure host work: works on a packing-only context. */
typedef struct ksh_taint { const char* key; const char* value; const char* effect; } ksh_taint;
int ksh_context_set_node_taints(ksh_context* ctx, const char* const* node_names, const uint64_t* taint_offset,
                                const ksh_taint* taints, uint64_t n);

/* Per-group tolerations and node affinity (pods of one group share them, as they share selectors).
 * Group g tolerates tolerations[toleration_offset[g] .. toleration_offset[g + 1]) (toleration_offset [G + 1] or NULL:
 * none), matched against each taint as upstream's ToleratesTaint: an empty effect matches every effect, an empty key
 * every key, operator Exists ignores the value, Equal or "" compares it.  Node-affinity term t of group term_owner[t] is
 * the AND of requirements[term_req_offset[t] .. term_req_offset[t + 1]); term_weight[t] 0 = a required term (ORed),
 * [1, 100] = a preferred one.  Requirement operators In, NotIn, Exists, DoesNotExist, Gt, Lt over the node store's label
 * values; NotIn and DoesNotExist match nodes without the key; Gt and Lt parse the node's value as a base-10 int64, and a
 * value that does not parse never matches.  KS_ERR_INVALID for what API validation rejects: an unknown toleration or
 * requirement operator, Exists with a value, In/NotIn without values, Gt/Lt without exactly one integer value,
 * Exists/DoesNotExist with values; KS_ERR_RANGE for more than 64 distinct taints in the store or more than
 * KS_NODE_RULES_MAX_KEYS requirement keys. */
typedef struct ksh_toleration { const char* key; const char* op; const char* value; const char* effect; } ksh_toleration;
typedef struct ksh_node_selector_requirement {
    const char* key;
    const char* op;                      /* In, NotIn, Exists, DoesNotExist, Gt, Lt */
    const char* const* values;
    uint32_t n_values;
} ksh_node_selector_requirement;
typedef struct ksh_node_rules {
    const uint64_t* toleration_offset;   /* [G + 1] or NULL */
    const ksh_toleration* tolerations;
    uint32_t n_terms;
    const int32_t* term_owner;           /* [T] */
    const uint32_t* term_weight;         /* [T] */
    const uint64_t* term_req_offset;     /* [T + 1] */
    const ksh_node_selector_requirement* requirements;
    uint32_t weight_taint;               /* default profile 3 */
    uint32_t weight_node_affinity;       /* default profile 2 */
} ksh_node_rules;

/* The compilation ksh_reconcile_nodes hands to ks_node_bind, evaluated per (group g, node n) at g * N + n from the
 * compiled masks and domain sets: out_hard = 1 when n carries a NoSchedule/NoExecute taint g does not tolerate,
 * out_affinity = 1 when n passes g's required node affinity, out_soft = n's PreferNoSchedule taints g does not tolerate
 * (by the tolerations whose effect is empty or PreferNoSchedule), out_preferred = the summed weights of g's preferred
 * terms n matches.  Each output may be NULL.  Errors as ksh_reconcile_nodes' compilation.  Pure host work: works on a
 * packing-only context. */
int ksh_compile_node_rules(ksh_context* ctx, uint32_t n_groups, const ksh_node_rules* rules, uint8_t* out_hard,
                           uint8_t* out_affinity, uint32_t* out_soft, uint32_t* out_preferred);

/* reconcile() under the default profile with taints and node affinity: ksh_reconcile_profile with the context's node
 * taints and `rules' (NULL: no toleration and no term), bound by ks_node_bind.  An unbound pod gets
 * KSH_RECONCILE_NODE_RULES_UNSATISFIED when some node fit it but taints or required node affinity refused every such
 * node, else the statuses map as in ksh_reconcile_affinity over the nodes that pass both.  Errors as
 * ksh_reconcile_profile, ks_node_bind and ksh_compile_node_rules. */
int ksh_reconcile_nodes(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, const int32_t* group,
                        uint32_t n_groups, const char* const* topology_keys, uint32_t n_keys,
                        const uint32_t* max_skew /* or NULL */, const uint32_t* min_domains,
                        const char* const* existing_node_names, const uint64_t* existing_offset,
                        const ksh_pod_affinity* aff /* or NULL */, const ks_bind_scoring* scoring,
                        const ksh_node_rules* rules /* or NULL */, int policy, int32_t* out_status,
                        int32_t* out_node_idx, char* json, size_t cap, int64_t* out_json_off);

/* Extended resources (ks_fit_bind, DESIGN.md 5r).  The context keeps, per node, the allocatable quantity of every name
 * other than cpu and memory (from ks_node_obj.allocatable), and per bound pod its non-zero requests of such names summed
 * over spec.containers, as it keeps cpu and memory; every node and pod event keeps them in step.  Quantities parse as
 * integers, as memory does.  A quantity that does not parse is recorded, not rejected, so no other call changes: the
 * calls below report it, naming the node or pod, only when the batch requests that resource: KS_ERR_PARSE for a
 * quantity that does not parse, KS_ERR_RANGE for a pod whose requests of one name sum past int64 over its containers.
 * A batch's resources: "pods" first, then every name other than cpu and memory that some pod of the batch requests with
 * a non-zero quantity, in order of first request; more than KS_BIND_MAX_RESOURCES is KS_ERR_RANGE (split the batch).
 * node_free[r * N + n] = node n's allocatable of resource r minus the requests of the pods bound there ("pods": minus
 * their number); a name missing from a node's allocatable counts as 0, as upstream, so a node without "pods" takes no
 * pod (callers that build synthetic nodes must list it).  pod_req[p * R + r] = pod p's request (1 for "pods").
 * ksh_compile_resources writes the names of the batch `pods` (taken whole, as the pods that go to the device) into
 * names (each NUL-terminated; KS_ERR_RANGE when they do not fit in cap), node_free [R * N] and pod_req [n_pods * R]
 * (either may be NULL; size them for R = KS_BIND_MAX_RESOURCES) and returns R.  Pure host work: works on a packing-only
 * context. */
int ksh_compile_resources(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, char* names, size_t cap,
                          int64_t* out_node_free, int64_t* out_pod_req);

/* reconcile() under the default profile with taints, node affinity and NodeResourcesFit's pod count and scalar
 * resources: ksh_reconcile_nodes' arguments, bound by ks_fit_bind over the batch's resources (the pods that go to the
 * device).  An unbound pod gets KSH_RECONCILE_INSUFFICIENT_RESOURCES when some node passed cpu, memory and selector but
 * every such node failed a resource, else the statuses of ksh_reconcile_nodes over the nodes that pass every resource.
 * Each bind is recorded with its extended requests, so the next call sees them.  Errors as ksh_reconcile_nodes,
 * ks_fit_bind and ksh_compile_resources. */
int ksh_reconcile_fit(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, const int32_t* group,
                      uint32_t n_groups, const char* const* topology_keys, uint32_t n_keys,
                      const uint32_t* max_skew /* or NULL */, const uint32_t* min_domains,
                      const char* const* existing_node_names, const uint64_t* existing_offset,
                      const ksh_pod_affinity* aff /* or NULL */, const ks_bind_scoring* scoring,
                      const ksh_node_rules* rules /* or NULL */, int policy, int32_t* out_status,
                      int32_t* out_node_idx, char* json, size_t cap, int64_t* out_json_off);

/* reconcile() for pod groups under the full bind filter (ks_gang_fit_bind, DESIGN.md 5s): ksh_reconcile_fit's arguments
 * plus gangs cut as ksh_reconcile_gangs cuts its groups.  Gang j is pods [gang_offset[j], gang_offset[j + 1]), at least
 * one pod, min_member[j] <= its size, and no other size limit than ks_gang_fit_bind's queue; its pods may belong to
 * different groups.  Members are filtered as ksh_reconcile_gangs filters them: already bound members are skipped
 * (KSH_RECONCILE_OK, node -1) and count toward min_member; nameless pods get KSH_RECONCILE_BINDING_OBJECT_FAILED and do
 * not count; the rest of each gang goes to the device with max(0, min_member - bound members).  The batch's resources
 * are built as ksh_compile_resources builds them over the pods that go to the device.  The pods of a gang that rolls
 * back, or that has fewer schedulable members than it still needs, get KSH_RECONCILE_GANG_UNSATISFIED: no Binding body,
 * and no charge or extended request is recorded for them.  The pods of a gang that commits get ksh_reconcile_fit's
 * statuses.  out_placed[n_gangs] (may be NULL) = the gang's pods the device placed before any rollback.  Offsets and
 * sizes are checked first: KS_ERR_INVALID (offsets) / KS_ERR_RANGE (an empty gang, min_member); otherwise errors as
 * ksh_reconcile_fit and ks_gang_fit_bind. */
int ksh_reconcile_fit_gangs(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, const int32_t* group,
                            uint32_t n_groups, const char* const* topology_keys, uint32_t n_keys,
                            const uint32_t* max_skew /* or NULL */, const uint32_t* min_domains,
                            const char* const* existing_node_names, const uint64_t* existing_offset,
                            const ksh_pod_affinity* aff /* or NULL */, const ks_bind_scoring* scoring,
                            const ksh_node_rules* rules /* or NULL */, const uint64_t* gang_offset, uint64_t n_gangs,
                            const uint32_t* min_member, int policy, int32_t* out_status, int32_t* out_node_idx,
                            uint32_t* out_placed, char* json, size_t cap, int64_t* out_json_off);

/* Priority preemption under the full filter over objects (ks_fit_preempt, DESIGN.md 5t): ksh_preempt_pods' arguments
 * plus group[n_pods] in [-1, n_groups) and rules (NULL allowed), as ksh_reconcile_nodes takes them.  The context's node
 * taints and the rules' tolerations and node-affinity terms are compiled as ksh_reconcile_nodes compiles them; the
 * batch's resources are built as ksh_compile_resources builds them over `pods`, and each bound pod's bound_req from its
 * recorded extended requests, 1 for "pods".  Bound pods without namespace and name are passed at priority INT32_MAX and
 * are never victims; victim keys are written as ksh_preempt_pods writes them.  A malformed quantity of a requested
 * resource is reported as ksh_reconcile_fit reports it (KS_ERR_PARSE or KS_ERR_RANGE, naming the node or pod).  Nothing
 * is charged.  KS_ERR_RANGE for max_victims outside [1, KS_PREEMPT_MAX_VICTIMS]; KS_ERR_NO_DEVICE on a packing-only
 * context. */
int ksh_preempt_fit_pods(ksh_context* ctx, const ks_pod_obj* pods, uint64_t n_pods, const int32_t* group,
                         uint32_t n_groups, const ksh_node_rules* rules /* or NULL */, const int32_t* pod_priority,
                         uint32_t max_victims, ks_preemption* out, char* victims, size_t cap, int64_t* out_victim_off);

/* Node drain under the full filter over objects (ks_fit_drain_check, DESIGN.md 5u): ksh_drain_nodes' arguments and
 * checks plus group[pod_offset[n]] in [-1, n_groups) and rules (NULL allowed), as ksh_preempt_fit_pods takes them.  The
 * context's node taints and the rules' tolerations and node-affinity terms are compiled as ksh_preempt_fit_pods compiles
 * them; the batch's resources are built as ksh_compile_resources builds them over the drained pods, so the pod count is
 * always among them and a destination at its allocatable "pods" takes no more ("Too many pods").  The drained pods are
 * bound to their candidate, which is never a destination, so the context's node_free is used as it is.
 * Cordoned and draining nodes: mark them with the taint node.kubernetes.io/unschedulable:NoSchedule through
 * ksh_context_set_node_taints, as the node lifecycle controller does; a group that does not tolerate it then sends
 * nothing there.  out_refused[4n] (or NULL) as ks_fit_drain_check gives it.  A malformed quantity of a requested
 * resource is reported as ksh_reconcile_fit reports it (KS_ERR_PARSE or KS_ERR_RANGE, naming the node or pod).  Nothing
 * is charged.  KS_ERR_NO_DEVICE on a packing-only context. */
int ksh_drain_fit_nodes(ksh_context* ctx, const char* const* node_names, uint64_t n, const ks_pod_obj* pods,
                        const uint64_t* pod_offset, const int32_t* group, uint32_t n_groups,
                        const ksh_node_rules* rules /* or NULL */, int policy, uint32_t flags, uint32_t* out_placed,
                        int32_t* out_node_idx, uint32_t* out_refused /* [4n] or NULL */);

/* Node-group scale-up estimate under the full filter over objects (ks_fit_scaleup_estimate, DESIGN.md 5v):
 * ksh_scaleup_estimate's arguments, checks and packing (templates, overhead pods, the call-local label dictionary) plus
 * group[n_pods] in [-1, n_groups) and rules (NULL allowed), as ksh_drain_fit_nodes takes them, and each template's
 * spec.taints: template t carries template_taints[template_taint_offset[t] .. template_taint_offset[t + 1])
 * (template_taint_offset [n_templates + 1] or NULL: none), checked as ksh_context_set_node_taints checks a node's.
 * Templates are not in the context's node store, so the rules are compiled over the templates: the taint bits from
 * their taints, and each node-affinity key's domains from their labels, numbered by first appearance in template order.
 * The resources are the batch's, as ksh_compile_resources builds them over `pods` ("pods" first), and a template's
 * node_free is its allocatable of each name (0 when missing, so a template without "pods" takes no pod, as upstream)
 * minus its overhead pods' requests and, for "pods", their number.  A malformed quantity of a requested resource is
 * reported as ksh_reconcile_fit reports it, naming the template or overhead pod.  The context's node store, bound list
 * and snapshot are not changed.  Outputs as ks_fit_scaleup_estimate gives them (out_used is not returned here).
 * KS_ERR_NO_DEVICE on a packing-only context, after every check. */
int ksh_scaleup_fit_estimate(ksh_context* ctx, const ks_node_obj* templates, uint64_t n_templates,
                             const uint32_t* max_nodes, const uint64_t* template_taint_offset /* [T + 1] or NULL */,
                             const ksh_taint* template_taints, const ks_pod_obj* overhead_pods, uint64_t n_overhead,
                             const ks_pod_obj* pods, uint64_t n_pods, const int32_t* group, uint32_t n_groups,
                             const ksh_node_rules* rules /* or NULL */, ks_scaleup_option* out, int32_t* out_best,
                             int32_t* out_node /* [T * n_pods] or NULL */, uint32_t* out_refused /* [4 n_pods] or NULL */);

#ifdef __cplusplus
}
#endif
#endif /* KSCHED_HOST_H */
