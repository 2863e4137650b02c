// ksched.rs — safe wrapper that keeps the reference's own signatures (SURVEY.md §8(b)):
//     check_node_validity(&Pod, &Node-index, &Gpu) -> Result<(), InvalidNodeReason>      src/predicates.rs:63-77
//     select_node_for_pod(&Pod, &Gpu) -> Option<node name>                               src/main.rs:51-71
//     reconcile body: Binding JSON for the POST                                          src/main.rs:79-103
// NOT COMPILED IN THIS REPOSITORY (no Rust toolchain in the build image); see ksched_sys.rs.
use std::ffi::{CStr, CString};
use std::os::raw::c_char;
use std::ptr;

use k8s_openapi::api::core::v1 as corev1;

use crate::ksched_sys::*;
use crate::predicates::InvalidNodeReason;

/// Owns the CStrings a `ks_pod_obj` view points into (the library copies what it keeps; views are per call).
pub struct PodView {
    _strings: Vec<CString>,
    _kvs: Vec<Vec<ks_kv>>,
    _containers: Vec<ks_container_obj>,
    pub obj: ks_pod_obj,
}

fn cs(v: &mut Vec<CString>, s: &str) -> *const c_char {
    v.push(CString::new(s).expect("NUL in a Kubernetes string"));
    v.last().unwrap().as_ptr()
}

impl PodView {
    pub fn new(pod: &corev1::Pod) -> PodView {
        let mut strings = Vec::new();
        let mut kvs: Vec<Vec<ks_kv>> = Vec::new();
        let mut containers = Vec::new();
        let ns = pod.metadata.namespace.as_deref().map(|s| cs(&mut strings, s)).unwrap_or(ptr::null());
        let name = pod.metadata.name.as_deref().map(|s| cs(&mut strings, s)).unwrap_or(ptr::null());
        let meta = cs(&mut strings, &serde_json::to_string(&pod.metadata).expect("ObjectMeta serialises"));
        let (mut node_name, mut has_sel, mut sel_ptr, mut n_sel) = (ptr::null(), 0, ptr::null(), 0u32);
        if let Some(spec) = &pod.spec {
            if let Some(nn) = &spec.node_name {
                node_name = cs(&mut strings, nn);
            }
            for c in &spec.containers {
                // only resources.requests is read (src/util.rs:58-62)
                match c.resources.as_ref().and_then(|r| r.requests.as_ref()) {
                    Some(req) => {
                        let v: Vec<ks_kv> = req.iter().map(|(k, q)| ks_kv { key: cs(&mut strings, k), val: cs(&mut strings, &q.0) }).collect();
                        kvs.push(v);
                        let v = kvs.last().unwrap();
                        containers.push(ks_container_obj { has_requests: 1, n_requests: v.len() as u32, requests: v.as_ptr() });
                    },
                    None => containers.push(ks_container_obj { has_requests: 0, n_requests: 0, requests: ptr::null() }),
                }
            }
            if let Some(sel) = &spec.node_selector {
                let v: Vec<ks_kv> = sel.iter().map(|(k, val)| ks_kv { key: cs(&mut strings, k), val: cs(&mut strings, val) }).collect();
                kvs.push(v);
                let v = kvs.last().unwrap();
                has_sel = 1;
                n_sel = v.len() as u32;
                sel_ptr = v.as_ptr();
            }
        }
        let obj = ks_pod_obj {
            ns,
            name,
            has_spec: pod.spec.is_some() as i32,
            node_name,
            n_containers: containers.len() as u32,
            containers: containers.as_ptr(),
            has_node_selector: has_sel,
            n_selector: n_sel,
            selector: sel_ptr,
            metadata_json: meta,
        };
        PodView { _strings: strings, _kvs: kvs, _containers: containers, obj }
    }
}

/// Owns the CStrings a `ks_node_obj` view points into (per call, as `PodView`).
pub struct NodeView {
    _strings: Vec<CString>,
    _kvs: Vec<Vec<ks_kv>>,
    pub obj: ks_node_obj,
}

impl NodeView {
    pub fn new(node: &corev1::Node) -> NodeView {
        let mut strings = Vec::new();
        let mut kvs: Vec<Vec<ks_kv>> = Vec::new();
        let name = node.metadata.name.as_deref().map(|s| cs(&mut strings, s)).unwrap_or(ptr::null());
        let (mut has_labels, mut n_labels, mut labels) = (0, 0u32, ptr::null());
        if let Some(l) = &node.metadata.labels {
            let v: Vec<ks_kv> = l.iter().map(|(k, val)| ks_kv { key: cs(&mut strings, k), val: cs(&mut strings, val) }).collect();
            kvs.push(v);
            let v = kvs.last().unwrap();
            (has_labels, n_labels, labels) = (1, v.len() as u32, v.as_ptr());
        }
        let (mut has_alloc, mut n_alloc, mut alloc) = (0, 0u32, ptr::null());
        if let Some(a) = node.status.as_ref().and_then(|s| s.allocatable.as_ref()) {
            let v: Vec<ks_kv> = a.iter().map(|(k, q)| ks_kv { key: cs(&mut strings, k), val: cs(&mut strings, &q.0) }).collect();
            kvs.push(v);
            let v = kvs.last().unwrap();
            (has_alloc, n_alloc, alloc) = (1, v.len() as u32, v.as_ptr());
        }
        let obj = ks_node_obj { name, has_labels, n_labels, labels, has_allocatable: has_alloc, n_allocatable: n_alloc,
                                allocatable: alloc };
        NodeView { _strings: strings, _kvs: kvs, obj }
    }
}

/// Replaces Context.node_store + the per-cell LIST (src/util.rs:12-15, src/predicates.rs:21-38).
pub struct Gpu {
    ctx: *mut ksh_context,
}
unsafe impl Send for Gpu {} // the library serialises per handle (one mutex per context)
unsafe impl Sync for Gpu {}

fn last_error() -> String {
    unsafe { CStr::from_ptr(ks_last_error()).to_string_lossy().into_owned() }
}

impl Gpu {
    pub fn new(device: i32) -> Result<Gpu, String> {
        let mut ctx = ptr::null_mut();
        if unsafe { ksh_context_create(device, &mut ctx) } != KS_OK {
            return Err(last_error());
        }
        Ok(Gpu { ctx })
    }

    /// src/predicates.rs:63-77 — same Result, same reason precedence (fit first, then selector)
    pub fn check_node_validity(&self, pod: &corev1::Pod, node_idx: u32) -> Result<(), InvalidNodeReason> {
        let v = PodView::new(pod);
        match unsafe { ksh_check_node_validity(self.ctx, &v.obj, node_idx) } {
            KS_CELL_OK => Ok(()),
            KS_CELL_NOT_ENOUGH_RESOURCES => Err(InvalidNodeReason::NotEnoughResources),
            KS_CELL_NODE_SELECTOR_MISMATCH => Err(InvalidNodeReason::NodeSelectorMismatch),
            e => panic!("ksh_check_node_validity failed ({}): {}", e, last_error()), // the reference panics on malformed objects too
        }
    }

    /// src/main.rs:51-71 — `None` when no node is feasible.  `reference_policy` keeps the <=ATTEMPTS random draws
    /// (seeded), otherwise the argmax of the leftover score over every feasible node.
    pub fn select_node_for_pod(&self, pod: &corev1::Pod, reference_policy: Option<(u64, u64)>) -> Option<String> {
        let v = PodView::new(pod);
        let mut idx: i32 = -1;
        let rc = match reference_policy {
            Some((seed, pod_counter)) => unsafe {
                ksh_select_node_for_pod(self.ctx, &v.obj, 1, KS_REFERENCE_ATTEMPTS, seed, pod_counter, &mut idx, ptr::null_mut(),
                                        ptr::null_mut(), ptr::null_mut())
            },
            None => unsafe { ksh_select_nodes(self.ctx, &v.obj, 1, KS_SCORE_LEFTOVER, &mut idx, ptr::null_mut(), ptr::null_mut()) },
        };
        if rc != KS_OK {
            panic!("select failed ({}): {}", rc, last_error());
        }
        if idx < 0 {
            return None;
        }
        Some(unsafe { CStr::from_ptr(ksh_context_node_name(self.ctx, idx as u32)) }.to_string_lossy().into_owned())
    }

    /// Up to `k` (1..=KS_TOPK_MAX) feasible nodes for the pod, best first: (node name, score) under the leftover score.
    /// The first is what `select_node_for_pod` picks; the rest are the fall-backs to try when its Binding POST fails.
    /// Nothing is charged: report the bind that succeeded with `ksh_context_pod_bound`.  Err = the library's status.
    pub fn rank_nodes(&self, pod: &corev1::Pod, k: u32) -> Result<Vec<(String, i64)>, i32> {
        let v = PodView::new(pod);
        let mut idx = vec![-1i32; k as usize];
        let mut score = vec![0i64; k as usize];
        let rc = unsafe {
            ksh_rank_nodes(self.ctx, &v.obj, 1, KS_SCORE_LEFTOVER, k, idx.as_mut_ptr(), score.as_mut_ptr(), ptr::null_mut())
        };
        if rc != KS_OK {
            return Err(rc);
        }
        Ok(idx.iter().zip(score.iter()).take_while(|(i, _)| **i >= 0).map(|(i, s)| {
            let name = unsafe { CStr::from_ptr(ksh_context_node_name(self.ctx, *i as u32)) }.to_string_lossy().into_owned();
            (name, *s)
        }).collect())
    }

    /// src/main.rs:79-103 up to (not including) the POST: Ok(Some(body)) = bind, Ok(None) = already bound,
    /// Err(1) = NoNodeFound, Err(2) = CreateBindingObjectFailed.  A failed POST needs no rollback call: the requeued
    /// pod comes back through reconcile(), which releases the earlier charge before it selects again.
    pub fn reconcile(&self, pod: &corev1::Pod) -> Result<Option<String>, i32> {
        let v = PodView::new(pod);
        let mut idx: i32 = -1;
        let mut buf = vec![0u8; 16384];
        match unsafe { ksh_reconcile(self.ctx, &v.obj, KS_SCORE_LEFTOVER, &mut idx, buf.as_mut_ptr() as *mut c_char, buf.len()) } {
            KSH_RECONCILE_OK if idx < 0 => Ok(None),
            KSH_RECONCILE_OK => Ok(Some(unsafe { CStr::from_ptr(buf.as_ptr() as *const c_char) }.to_string_lossy().into_owned())),
            e => Err(e),
        }
    }

    /// Why a pod did not schedule: the per-check rejection counts and, when no node is feasible, the FailedScheduling
    /// message (`0/5 nodes are available: 2 Insufficient cpu, ...`) that `kubectl describe pod` would show.
    pub fn explain(&self, pod: &corev1::Pod) -> (ks_pod_reasons, Option<String>) {
        let v = PodView::new(pod);
        let mut r = ks_pod_reasons::default();
        let mut buf = vec![0u8; 512];
        let mut off: i64 = -1;
        let rc = unsafe { ksh_explain_pods(self.ctx, &v.obj, 1, &mut r, buf.as_mut_ptr() as *mut c_char, buf.len(), &mut off) };
        if rc != KS_OK {
            panic!("ksh_explain_pods failed ({}): {}", rc, last_error());
        }
        let msg = if off < 0 {
            None
        } else {
            Some(unsafe { CStr::from_ptr(buf.as_ptr().add(off as usize) as *const c_char) }.to_string_lossy().into_owned())
        };
        (r, msg)
    }

    /// Priority preemption for a pod no node accepts (upstream's PostFilter without PodDisruptionBudgets): the node
    /// name and the "namespace/name" keys of the lower-priority pods to evict there, in visit order; None = no plan.
    /// `priority` is the pod's spec.priority; bound pods' priorities come from `ksh_context_set_pod_priorities`.
    /// Nothing is charged: DELETE the victims, report each with `ksh_context_pod_deleted`, requeue the pod.
    pub fn preempt(&self, pod: &corev1::Pod, priority: i32, max_victims: u32) -> Result<Option<(String, Vec<String>)>, i32> {
        let v = PodView::new(pod);
        let mut row = ks_preemption::default();
        let mut buf = vec![0u8; 256 * max_victims as usize];
        let mut off: i64 = -1;
        let rc = unsafe {
            ksh_preempt_pods(self.ctx, &v.obj, 1, &priority, max_victims, &mut row, buf.as_mut_ptr() as *mut c_char,
                             buf.len(), &mut off)
        };
        if rc != KS_OK {
            return Err(rc);
        }
        if row.node_idx < 0 || off < 0 {
            return Ok(None);
        }
        let node = unsafe { CStr::from_ptr(ksh_context_node_name(self.ctx, row.node_idx as u32)) }.to_string_lossy().into_owned();
        let mut keys = Vec::with_capacity(row.n_victims as usize);
        let mut at = off as usize;
        for _ in 0..row.n_victims {
            let k = unsafe { CStr::from_ptr(buf.as_ptr().add(at) as *const c_char) };
            at += k.to_bytes().len() + 1;
            keys.push(k.to_string_lossy().into_owned());
        }
        Ok(Some((node, keys)))
    }

    /// Pod groups, all or nothing (upstream coscheduling's PodGroup `minMember`): `groups` holds each group's pods
    /// and min_member, in order.  Per pod: Ok(Some(body)) = bind, Ok(None) = already bound (counts toward its group),
    /// Err(1) = NoNodeFound in a group that committed, Err(2) = CreateBindingObjectFailed, Err(4) = the group rolled
    /// back (nothing charged).  Outer Err = the library's status (bad offsets or sizes, no device).
    pub fn reconcile_gangs(&self, groups: &[(&[corev1::Pod], u32)]) -> Result<Vec<Result<Option<String>, i32>>, i32> {
        let views: Vec<PodView> = groups.iter().flat_map(|(pods, _)| pods.iter().map(PodView::new)).collect();
        // ks_pod_obj is plain pointers into `views`, which outlive the call
        let objs: Vec<ks_pod_obj> = views.iter().map(|v| unsafe { ptr::read(&v.obj) }).collect();
        let mut offset = vec![0u64];
        for (pods, _) in groups {
            offset.push(offset.last().unwrap() + pods.len() as u64);
        }
        let min_member: Vec<u32> = groups.iter().map(|(_, m)| *m).collect();
        let n = objs.len();
        let (mut status, mut idx, mut off) = (vec![0i32; n], vec![-1i32; n], vec![-1i64; n]);
        // room for every body: {"apiVersion":"v1","kind":"Binding","metadata":<ObjectMeta JSON>,"target":{"name":"<node>"}}
        // with the longest node name JSON-escaped at worst 6 bytes per character, and the NUL
        let longest_node = (0..unsafe { ksh_context_num_nodes(self.ctx) })
            .map(|k| unsafe { CStr::from_ptr(ksh_context_node_name(self.ctx, k)) }.to_bytes().len())
            .max()
            .unwrap_or(0);
        let cap: usize = views.iter()
            .map(|v| unsafe { CStr::from_ptr(v.obj.metadata_json) }.to_bytes().len() + 6 * longest_node + 128)
            .sum();
        let mut buf = vec![0u8; cap.max(1)];
        let rc = unsafe {
            ksh_reconcile_gangs(self.ctx, objs.as_ptr(), n as u64, offset.as_ptr(), groups.len() as u64, min_member.as_ptr(),
                                KS_SCORE_LEFTOVER, status.as_mut_ptr(), idx.as_mut_ptr(), ptr::null_mut(),
                                buf.as_mut_ptr() as *mut c_char, buf.len(), off.as_mut_ptr())
        };
        if rc != KS_OK {
            return Err(rc);
        }
        Ok((0..n).map(|i| match status[i] {
            KSH_RECONCILE_OK if idx[i] < 0 => Ok(None), // already running
            // bound and charged: the buffer holds every body, so a missing one is a broken invariant, not a skip
            KSH_RECONCILE_OK if off[i] < 0 => panic!("ksh_reconcile_gangs bound pod {} but returned no Binding body", i),
            KSH_RECONCILE_OK => Ok(Some(unsafe { CStr::from_ptr(buf.as_ptr().add(off[i] as usize) as *const c_char) }
                .to_string_lossy().into_owned())),
            e => Err(e),
        }).collect())
    }

    /// Node drain / scale-down check (cluster-autoscaler's removal simulation): `candidates` holds each node's name and
    /// the pods to move off it (its bound pods, after the caller's PodDisruptionBudget / DaemonSet / local-storage
    /// filtering).  Each candidate is evaluated on its own against the current cluster; nothing is charged.  Per
    /// candidate: Some(destination node names, one per pod) when every pod finds a place, None when it cannot be
    /// drained.  `exclude_candidates`: no listed node takes pods from another (several nodes removed together).
    pub fn drain_nodes(&self, candidates: &[(&str, &[corev1::Pod])], exclude_candidates: bool)
                       -> Result<Vec<Option<Vec<String>>>, i32> {
        let names: Vec<CString> = candidates.iter().map(|(n, _)| CString::new(*n).expect("NUL in a node name")).collect();
        let name_ptrs: Vec<*const c_char> = names.iter().map(|n| n.as_ptr()).collect();
        let views: Vec<PodView> = candidates.iter().flat_map(|(_, pods)| pods.iter().map(PodView::new)).collect();
        let objs: Vec<ks_pod_obj> = views.iter().map(|v| unsafe { ptr::read(&v.obj) }).collect();
        let mut offset = vec![0u64];
        for (_, pods) in candidates {
            offset.push(offset.last().unwrap() + pods.len() as u64);
        }
        let mut placed = vec![0u32; candidates.len()];
        let mut idx = vec![-1i32; objs.len()];
        let flags = if exclude_candidates { KS_DRAIN_EXCLUDE_CANDIDATES } else { 0 };
        let rc = unsafe {
            ksh_drain_nodes(self.ctx, name_ptrs.as_ptr(), candidates.len() as u64, objs.as_ptr(), offset.as_ptr(),
                            KS_SCORE_LEFTOVER, flags, placed.as_mut_ptr(), idx.as_mut_ptr())
        };
        if rc != KS_OK {
            return Err(rc);
        }
        Ok((0..candidates.len()).map(|d| {
            let (a, b) = (offset[d] as usize, offset[d + 1] as usize);
            if placed[d] as usize != b - a {
                return None;
            }
            Some(idx[a..b].iter().map(|&n| unsafe { CStr::from_ptr(ksh_context_node_name(self.ctx, n as u32)) }
                .to_string_lossy().into_owned()).collect())
        }).collect())
    }
}

/// One node template of a node group for `Gpu::scaleup_estimate_packed`: allocatable, capacity of an empty node (allocatable
/// minus its DaemonSet and system pods), label words in the call's own bit layout, and the nodes the group may add.
pub struct NodeTemplate {
    pub alloc_cpu: i64,
    pub alloc_mem: i64,
    pub free_cpu: i64,
    pub free_mem: i64,
    pub labels: Vec<u64>,
    pub max_nodes: u32,
}

impl Gpu {
    /// Node-group scale-up estimate (cluster-autoscaler's binpacking estimator) over objects: each template is a Node
    /// object standing for one new node of a group (labels it would carry, instance type included; allocatable) with
    /// the nodes the group may still add; `daemonsets` are the pods that would run on every such node, each with
    /// spec.nodeName set to its template's name; `pending` are the pods no node accepts.  Each template is packed on its
    /// own by first fit in decreasing-size order; nothing is charged.  Returns the per-template rows, the best template
    /// (most pods placed, then utilization, then fewest nodes) and, per (template, pending pod), the new node's ordinal
    /// or -1.  Err = the library's status (KS_ERR_NO_DEVICE on a packing-only context).
    pub fn scaleup_estimate(&self, templates: &[(corev1::Node, u32)], daemonsets: &[corev1::Pod], pending: &[corev1::Pod])
                            -> Result<(Vec<ks_scaleup_option>, Option<usize>, Vec<i32>), i32> {
        let tv: Vec<NodeView> = templates.iter().map(|(n, _)| NodeView::new(n)).collect();
        let tobj: Vec<ks_node_obj> = tv.iter().map(|v| unsafe { ptr::read(&v.obj) }).collect();
        let max_nodes: Vec<u32> = templates.iter().map(|(_, m)| *m).collect();
        let dv: Vec<PodView> = daemonsets.iter().map(PodView::new).collect();
        let dobj: Vec<ks_pod_obj> = dv.iter().map(|v| unsafe { ptr::read(&v.obj) }).collect();
        let pv: Vec<PodView> = pending.iter().map(PodView::new).collect();
        let pobj: Vec<ks_pod_obj> = pv.iter().map(|v| unsafe { ptr::read(&v.obj) }).collect();
        let mut rows = vec![ks_scaleup_option::default(); templates.len()];
        let mut best = -1i32;
        let mut node = vec![-1i32; templates.len() * pending.len()];
        let rc = unsafe {
            ksh_scaleup_estimate(self.ctx, tobj.as_ptr(), tobj.len() as u64, max_nodes.as_ptr(), dobj.as_ptr(),
                                 dobj.len() as u64, pobj.as_ptr(), pobj.len() as u64, rows.as_mut_ptr(), &mut best,
                                 node.as_mut_ptr(), ptr::null_mut())
        };
        if rc != KS_OK {
            return Err(rc);
        }
        Ok((rows, if best < 0 { None } else { Some(best as usize) }, node))
    }

    /// The same over packed pods, for callers with their own label bit layout: `req` holds each pending pod's (cpu
    /// millicores, memory bytes) and `sel` its `label_words` selector words, in the templates' bit layout.  Panics when
    /// `sel` or a template's `labels` does not hold `label_words` words per entry.
    pub fn scaleup_estimate_packed(&self, req: &[(i64, i64)], sel: &[u64], label_words: u32, templates: &[NodeTemplate])
                                   -> Result<(Vec<ks_scaleup_option>, Option<usize>, Vec<i32>), i32> {
        let w = label_words as usize;
        assert_eq!(sel.len(), req.len() * w, "sel must hold label_words words per pod");
        assert!(templates.iter().all(|t| t.labels.len() == w), "each template's labels must hold label_words words");
        let snap = unsafe { ksh_context_snapshot(self.ctx) };
        if snap.is_null() {
            return Err(KS_ERR_NO_DEVICE);
        }
        let cpu: Vec<i64> = req.iter().map(|r| r.0).collect();
        let mem: Vec<i64> = req.iter().map(|r| r.1).collect();
        let ac: Vec<i64> = templates.iter().map(|t| t.alloc_cpu).collect();
        let am: Vec<i64> = templates.iter().map(|t| t.alloc_mem).collect();
        let fc: Vec<i64> = templates.iter().map(|t| t.free_cpu).collect();
        let fm: Vec<i64> = templates.iter().map(|t| t.free_mem).collect();
        let labels: Vec<u64> = templates.iter().flat_map(|t| t.labels.iter().copied()).collect();
        let max_nodes: Vec<u32> = templates.iter().map(|t| t.max_nodes).collect();
        let pods = ks_pods { n: req.len() as u64, req_cpu: cpu.as_ptr(), req_mem: mem.as_ptr(), sel: sel.as_ptr(),
                             mem_space: KS_MEM_HOST };
        let t = ks_node_templates { n: templates.len() as u64, label_words, alloc_cpu: ac.as_ptr(), alloc_mem: am.as_ptr(),
                                    free_cpu: fc.as_ptr(), free_mem: fm.as_ptr(), labels: labels.as_ptr(),
                                    max_nodes: max_nodes.as_ptr() };
        let mut rows = vec![ks_scaleup_option::default(); templates.len()];
        let mut best = -1i32;
        let mut node = vec![-1i32; templates.len() * req.len()];
        let rc = unsafe {
            ks_scaleup_estimate(snap, &pods, &t, rows.as_mut_ptr(), &mut best, node.as_mut_ptr(), ptr::null_mut())
        };
        if rc != KS_OK {
            return Err(rc);
        }
        Ok((rows, if best < 0 { None } else { Some(best as usize) }, node))
    }
}

impl Gpu {
    /// Replica placement (a Deployment, ReplicaSet or Job scaled out; kubernetes-sigs/cluster-capacity): for each
    /// (pod, replicas) pair, where that many copies of the pod would land placed one after another by the library's
    /// argmax, with the earlier copies bound, and the row with the cluster's capacity for the pod.  Nothing is charged.
    /// Returns per pair the row and the node names of the placed copies in placement order (shorter than the request
    /// when the capacity is).  Err = the library's status (KS_ERR_NO_DEVICE on a packing-only context).  `policy`:
    /// KS_SCORE_LEFTOVER, KS_SCORE_LEAST_ALLOCATED, KS_SCORE_MOST_ALLOCATED (bin-packing: fills busy nodes first) or
    /// KS_SCORE_LEAST_BALANCED (the default scheduler's choice; its copies are placed one at a time).
    pub fn place_replicas(&self, specs: &[(corev1::Pod, u32)], policy: i32)
                          -> Result<Vec<(ks_replica_plan, Vec<String>)>, i32> {
        let pv: Vec<PodView> = specs.iter().map(|(p, _)| PodView::new(p)).collect();
        let pobj: Vec<ks_pod_obj> = pv.iter().map(|v| unsafe { ptr::read(&v.obj) }).collect();
        let replicas: Vec<u32> = specs.iter().map(|(_, r)| *r).collect();
        let total: usize = replicas.iter().map(|&r| r as usize).sum();
        let mut rows = vec![ks_replica_plan::default(); specs.len()];
        let mut node = vec![-1i32; total];
        let rc = unsafe {
            ksh_place_replicas(self.ctx, pobj.as_ptr(), pobj.len() as u64, replicas.as_ptr(), policy, rows.as_mut_ptr(),
                               node.as_mut_ptr(), ptr::null_mut())
        };
        if rc != KS_OK {
            return Err(rc);
        }
        let mut at = 0usize;
        Ok(rows.into_iter().zip(replicas).map(|(row, r)| {
            let names = node[at..at + row.placed as usize].iter().map(|&n| unsafe {
                CStr::from_ptr(ksh_context_node_name(self.ctx, n as u32)) }.to_string_lossy().into_owned()).collect();
            at += r as usize;
            (row, names)
        }).collect())
    }

    /// Replica placement under one topology spread constraint (`topologySpreadConstraints` with `whenUnsatisfiable:
    /// DoNotSchedule`): as `place_replicas`, but the copies spread over the values of `topology_key` (e.g.
    /// "topology.kubernetes.io/zone" or "kubernetes.io/hostname") within `max_skew` of the least-loaded eligible
    /// domain; `existing[t]` names the nodes of the bound pods that match spec t's constraint selector.  Returns per
    /// spec the row (`blocked_domain` indexes the returned domain values) and the node names of the placed copies, and
    /// the domain values.  Nothing is charged.
    pub fn place_replicas_spread(&self, specs: &[(corev1::Pod, u32, u32)], topology_key: &str, existing: &[Vec<String>],
                                 policy: i32) -> Result<(Vec<(ks_spread_plan, Vec<String>)>, Vec<String>), i32> {
        let key = CString::new(topology_key).map_err(|_| KS_ERR_INVALID)?;
        let n_nodes = unsafe { ksh_context_num_nodes(self.ctx) } as usize;
        let mut dom = vec![-1i32; n_nodes.max(1)];
        let mut d = 0u32;
        let mut names = vec![0 as c_char; 64 * n_nodes.max(1)];
        let mut off = vec![-1i64; n_nodes.max(1)];
        let rc = unsafe {
            ksh_context_topology_domains(self.ctx, key.as_ptr(), dom.as_mut_ptr(), &mut d, names.as_mut_ptr(), names.len(),
                                         off.as_mut_ptr())
        };
        if rc != KS_OK {
            return Err(rc);
        }
        let values: Vec<String> = off[..d as usize].iter().map(|&o| if o < 0 { String::new() } else {
            unsafe { CStr::from_ptr(names.as_ptr().add(o as usize)) }.to_string_lossy().into_owned() }).collect();
        let pv: Vec<PodView> = specs.iter().map(|(p, _, _)| PodView::new(p)).collect();
        let pobj: Vec<ks_pod_obj> = pv.iter().map(|v| unsafe { ptr::read(&v.obj) }).collect();
        let replicas: Vec<u32> = specs.iter().map(|s| s.1).collect();
        let skew: Vec<u32> = specs.iter().map(|s| s.2).collect();
        let mut ex: Vec<CString> = Vec::new();
        let mut ex_off = vec![0u64; specs.len() + 1];
        for t in 0..specs.len() {
            for name in existing.get(t).map(|v| v.as_slice()).unwrap_or(&[]) {
                ex.push(CString::new(name.as_str()).map_err(|_| KS_ERR_INVALID)?);
            }
            ex_off[t + 1] = ex.len() as u64;
        }
        let ex_ptr: Vec<*const c_char> = ex.iter().map(|s| s.as_ptr()).collect();
        let total: usize = replicas.iter().map(|&r| r as usize).sum();
        let mut rows = vec![ks_spread_plan::default(); specs.len()];
        let mut node = vec![-1i32; total];
        let rc = unsafe {
            ksh_place_replicas_spread(self.ctx, pobj.as_ptr(), pobj.len() as u64, replicas.as_ptr(), key.as_ptr(),
                                      skew.as_ptr(), ptr::null(), ex_ptr.as_ptr(), ex_off.as_ptr(), policy,
                                      rows.as_mut_ptr(), node.as_mut_ptr(), ptr::null_mut(), ptr::null_mut())
        };
        if rc != KS_OK {
            return Err(rc);
        }
        let mut at = 0usize;
        let plans = rows.into_iter().zip(replicas).map(|(row, r)| {
            let names = node[at..at + row.placed as usize].iter().map(|&n| unsafe {
                CStr::from_ptr(ksh_context_node_name(self.ctx, n as u32)) }.to_string_lossy().into_owned()).collect();
            at += r as usize;
            (row, names)
        }).collect();
        Ok((plans, values))
    }
}

impl Drop for Gpu {
    fn drop(&mut self) {
        unsafe { ksh_context_destroy(self.ctx) }
    }
}
