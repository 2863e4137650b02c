/* reconcile_loop.c — the reference's control flow (main.rs: reconcile per pod, /root/reference/src/main.rs:73-120)
 * driven through libksched.so from plain C, the way a Rust host would through the extern "C" block of
 * INTEGRATION.md.  The cluster is the hand-derived C1 vector of SURVEY.md §8c (5 nodes, 10 pods).
 *
 *   gcc -std=c99 -Iinclude examples/reconcile_loop.c -Lkube-scheduler-rs-reference_b200 -lksched \
 *       -Wl,-rpath,$PWD/kube-scheduler-rs-reference_b200 -o /tmp/reconcile_loop && /tmp/reconcile_loop [--sampling SEED | --batch]
 *
 * Without an H100 the library refuses to compute (no CPU fallback): the program prints the error and exits 3.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "ksched_host.h"

#define KV(k, v) {k, v}
#define N_NODES 5
#define N_BOUND 5
#define N_PODS 10

static int die(const char* what, int rc) {
    fprintf(stderr, "%s failed: %d (%s)\n", what, rc, ks_last_error());
    return 3;
}

int main(int argc, char** argv) {
    const int sampling = argc > 1 && strcmp(argv[1], "--sampling") == 0;
    const int batch = argc > 1 && strcmp(argv[1], "--batch") == 0;
    const uint64_t seed = argc > 2 ? strtoull(argv[2], NULL, 0) : 1;

    /* node store: what reflector::Store<Node>::state() holds (main.rs:56) */
    static const ks_kv a0[] = {KV("cpu", "4"), KV("memory", "8589934592")};
    static const ks_kv a1[] = {KV("cpu", "2"), KV("memory", "4294967296")};
    static const ks_kv a2[] = {KV("cpu", "8"), KV("memory", "17179869184")};
    static const ks_kv a3[] = {KV("cpu", "1"), KV("memory", "1073741824")};
    static const ks_kv zone_a[] = {KV("zone", "a")};
    static const ks_kv zone_b[] = {KV("zone", "b")};
    const ks_node_obj nodes[N_NODES] = {
        {"n0", 1, 1, zone_a, 1, 2, a0}, {"n1", 1, 1, zone_b, 1, 2, a1}, {"n2", 1, 1, zone_a, 1, 2, a2},
        {"n3", 0, 0, NULL, 1, 2, a3},   {"n4", 0, 0, NULL, 0, 0, NULL}, /* status = None -> available (0,0) */
    };

    /* pods already bound (what the LIST of predicates.rs:21-34 returns per node) */
    static const ks_kv r_b1[] = {KV("cpu", "500m"), KV("memory", "1073741824")};
    static const ks_kv r_b2[] = {KV("cpu", "2"), KV("memory", "4294967296")};
    static const ks_kv r_b3[] = {KV("cpu", "250m"), KV("memory", "268435456")};
    static const ks_kv r_b4[] = {KV("cpu", "1"), KV("memory", "1073741824")};
    static const ks_kv r_b5[] = {KV("cpu", "100m"), KV("memory", "1")};
    const ks_container_obj c_b1[] = {{1, 2, r_b1}}, c_b2[] = {{1, 2, r_b2}}, c_b3[] = {{1, 2, r_b3}, {1, 2, r_b3}},
                           c_b4[] = {{1, 2, r_b4}}, c_b5[] = {{1, 2, r_b5}};
    const ks_pod_obj bound[N_BOUND] = {
        {"default", "b1", 1, "n1", 1, c_b1, 0, 0, NULL, NULL}, {"default", "b2", 1, "n2", 1, c_b2, 0, 0, NULL, NULL},
        {"default", "b3", 1, "n2", 2, c_b3, 0, 0, NULL, NULL}, {"default", "b4", 1, "n3", 1, c_b4, 0, 0, NULL, NULL},
        {"default", "b5", 1, "n4", 1, c_b5, 0, 0, NULL, NULL},
    };

    /* pending pods (the Controller's queue) */
    static const ks_kv r1[] = {KV("cpu", "500m"), KV("memory", "1073741824")};
    static const ks_kv r2[] = {KV("cpu", "1500m"), KV("memory", "3221225472")};
    static const ks_kv r3[] = {KV("cpu", "1501m"), KV("memory", "1")};
    static const ks_kv r4[] = {KV("cpu", "100m"), KV("memory", "3221225473")};
    static const ks_kv r5[] = {KV("cpu", "4"), KV("memory", "8589934592")};
    static const ks_kv r6[] = {KV("cpu", "5500m"), KV("memory", "12348030976")};
    static const ks_kv r7a[] = {KV("cpu", "2"), KV("memory", "4294967296")};
    static const ks_kv r7b[] = {KV("cpu", "3500m"), KV("memory", "8053063680")};
    static const ks_kv r8[] = {KV("cpu", "5501m"), KV("memory", "0")};
    const ks_container_obj c1[] = {{1, 2, r1}}, c2[] = {{1, 2, r2}}, c3[] = {{1, 2, r3}}, c4[] = {{1, 2, r4}},
                           c5[] = {{1, 2, r5}}, c6[] = {{1, 2, r6}}, c7[] = {{1, 2, r7a}, {1, 2, r7b}},
                           c8[] = {{1, 2, r8}}, c9[] = {{0, 0, NULL}}; /* limits only: no requests */
    const ks_pod_obj pods[N_PODS] = {
        {"default", "p0", 1, NULL, 0, NULL, 0, 0, NULL, NULL},     {"default", "p1", 1, NULL, 1, c1, 1, 1, zone_a, NULL},
        {"default", "p2", 1, NULL, 1, c2, 0, 0, NULL,
         "{\"name\":\"p2\",\"namespace\":\"default\",\"uid\":\"0b5e\",\"labels\":{\"app\":\"web\"}}"},       {"default", "p3", 1, NULL, 1, c3, 0, 0, NULL, NULL},
        {"default", "p4", 1, NULL, 1, c4, 1, 1, zone_b, NULL},     {"default", "p5", 1, NULL, 1, c5, 0, 0, NULL, NULL},
        {"default", "p6", 1, NULL, 1, c6, 0, 0, NULL, NULL},       {"default", "p7", 1, NULL, 2, c7, 0, 0, NULL, NULL},
        {"default", "p8", 1, NULL, 1, c8, 0, 0, NULL, NULL},       {"default", "p9", 1, "n0", 1, c9, 0, 0, NULL, NULL}, /* already bound */
    };

    ksh_context* ctx = NULL;
    int rc = ksh_context_create(0, &ctx);
    if (rc) return die("ksh_context_create", rc);
    if ((rc = ksh_context_set_nodes(ctx, nodes, N_NODES))) return die("ksh_context_set_nodes", rc);
    if ((rc = ksh_context_set_cluster_pods(ctx, bound, N_BOUND))) return die("ksh_context_set_cluster_pods", rc);

    if (batch) { /* the whole queue in one call: one pack, the device's micro-batch loop, one Binding body per bound pod */
        int32_t status[N_PODS], node[N_PODS];
        int64_t off[N_PODS];
        static char bodies[N_PODS * 512];
        uint32_t rounds = 0;
        rc = ksh_reconcile_batch(ctx, pods, N_PODS, KS_SCORE_LEFTOVER, status, node, bodies, sizeof(bodies), off, &rounds);
        if (rc) return die("ksh_reconcile_batch", rc);
        for (int i = 0; i < N_PODS; i++)
            printf("%s: status %d %s\n", pods[i].name, status[i], off[i] >= 0 ? bodies + off[i] : "(no binding)");
        printf("%u round(s)\n", rounds);
        ksh_context_destroy(ctx);
        return 0;
    }
    for (int i = 0; i < N_PODS; i++) {
        int32_t node = -1;
        char body[512] = "";
        if (sampling && !ksh_is_pod_bound(&pods[i])) {
            /* the reference's own policy: <= 5 random draws, first valid node wins (main.rs:49-71) */
            uint32_t used = 0;
            int32_t draw_node[KS_REFERENCE_ATTEMPTS];
            uint8_t draw_code[KS_REFERENCE_ATTEMPTS];
            rc = ksh_select_node_for_pod(ctx, &pods[i], 1, KS_REFERENCE_ATTEMPTS, seed, (uint64_t)i, &node, &used, draw_node,
                                         draw_code);
            if (rc) return die("ksh_select_node_for_pod", rc);
            printf("%s: %u draws ->", pods[i].name, used);
            for (uint32_t k = 0; k < used; k++) printf(" %s(code %u)", ksh_context_node_name(ctx, (uint32_t)draw_node[k]), draw_code[k]);
            printf(" => %s\n", node >= 0 ? ksh_context_node_name(ctx, (uint32_t)node) : "NoNodeFound");
            continue;
        }
        rc = ksh_reconcile(ctx, &pods[i], KS_SCORE_LEFTOVER, &node, body, sizeof(body));
        if (rc < 0) return die("ksh_reconcile", rc);
        if (rc == KSH_RECONCILE_NO_NODE_FOUND) {
            printf("%s: ReconcileError::NoNodeFound\n", pods[i].name);
            /* why: the FailedScheduling message `kubectl describe pod` would show */
            ks_pod_reasons why;
            char msg[256];
            int64_t msg_off = -1;
            rc = ksh_explain_pods(ctx, &pods[i], 1, &why, msg, sizeof(msg), &msg_off);
            if (rc) return die("ksh_explain_pods", rc);
            if (msg_off >= 0) printf("%s: %s\n", pods[i].name, msg + msg_off);
        } else if (node < 0)
            printf("%s: already bound, skipped\n", pods[i].name);
        else
            printf("%s: POST /api/v1/namespaces/%s/pods/%s/binding %s\n", pods[i].name, pods[i].ns, pods[i].name, body);
    }
    ksh_context_destroy(ctx);
    return 0;
}
