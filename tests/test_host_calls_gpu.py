"""String-list outputs of the object-level calls that need ks_explain, ks_preempt and ks_gang_bind, under a buffer that
holds all entries, none, or one shorter entry after a longer one that is skipped (test_host_calls.py covers
ksh_reconcile_batch and ksh_context_topology_domains)."""
import pytest

from helpers import string_list_cases

pytestmark = pytest.mark.gpu


def test_explain_messages_under_a_small_buffer(ks):
    arena = ks.objects.ObjectArena()
    nodes = arena.nodes([{"name": f"n{i}", "labels": {"zone": "a"}, "allocatable": {"cpu": "2", "memory": "4Gi"}}
                         for i in range(3)])
    pods = arena.pods([{"name": "both", "ns": "d", "containers": [{"cpu": "9", "memory": "9Gi"}]},
                       {"name": "fits", "ns": "d", "containers": [{"cpu": "1"}]},
                       {"name": "cpu", "ns": "d", "containers": [{"cpu": "9"}]},
                       {"name": "selector", "ns": "d", "containers": [], "selector": {"zone": "b"}}])
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, 3)
        _, full = ctx.explain_pods(pods, 4)
        assert full == ["0/3 nodes are available: 3 Insufficient cpu, 3 Insufficient memory.", None,
                        "0/3 nodes are available: 3 Insufficient cpu.",
                        "0/3 nodes are available: 3 node(s) didn't match Pod's node affinity/selector."]
        for cap, want in string_list_cases(full):
            why, msgs = ctx.explain_pods(pods, 4, msg_cap=cap)
            assert msgs == want, cap
            assert why[:, 2].tolist() == [3, 0, 3, 0]  # the counts come back whatever the buffer holds


def test_preempt_victims_under_a_small_buffer(ks):
    arena = ks.objects.ObjectArena()
    nodes = arena.nodes([{"name": "n0", "labels": {"zone": "a"}, "allocatable": {"cpu": "2", "memory": "4Gi"}},
                         {"name": "n1", "labels": {"zone": "b"}, "allocatable": {"cpu": "2", "memory": "4Gi"}}])
    bound_s = [{"name": "first-victim", "ns": "d", "node_name": "n0", "containers": [{"cpu": "1"}]},
               {"name": "second-victim", "ns": "d", "node_name": "n0", "containers": [{"cpu": "1"}]},
               {"name": "c", "ns": "d", "node_name": "n1", "containers": [{"cpu": "2"}]}]
    bound = arena.pods(bound_s)
    pods = arena.pods([{"name": "q0", "ns": "d", "containers": [{"cpu": "2"}], "selector": {"zone": "a"}},
                       {"name": "q1", "ns": "d", "containers": [{"cpu": "1"}], "selector": {"zone": "z"}},
                       {"name": "q2", "ns": "d", "containers": [{"cpu": "1"}], "selector": {"zone": "b"}}])
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, 2)
        ctx.set_cluster_pods(bound, 3)
        ctx.set_pod_priorities(bound, [0, 0, 0], 3)
        _, full = ctx.preempt_pods(pods, 3, [10, 10, 10], 4)
        assert [None if v is None else sorted(v) for v in full] == [["d/first-victim", "d/second-victim"], None, ["d/c"]]
        for cap, want in string_list_cases(full, size=lambda keys: sum(len(k.encode()) + 1 for k in keys)):
            rows, victims = ctx.preempt_pods(pods, 3, [10, 10, 10], 4, victims_cap=cap)
            assert victims == want, cap
            assert rows["n_victims"].tolist() == [2, 0, 1]


def test_gang_bodies_under_a_small_buffer(ks):
    arena = ks.objects.ObjectArena()
    nodes = arena.nodes([{"name": "n0", "allocatable": {"cpu": "8", "memory": "8Gi"}}])
    pods_s = [{"name": "long", "ns": "d", "containers": [{"cpu": "1"}],
               "metadata_json": '{"name":"long","namespace":"d","labels":{"app":"' + "x" * 80 + '"}}'},
              {"name": "s", "ns": "d", "containers": [{"cpu": "1"}]},
              {"name": "bound", "ns": "d", "node_name": "n0", "containers": []},
              {"name": "mid", "ns": "d", "containers": [{"cpu": "1"}]}]
    full, cases = None, None
    for step in range(4):
        with ks.host.Context(0) as ctx:
            ctx.set_nodes(nodes, 1)
            ctx.set_cluster_pods(arena.pods([]), 0)
            cap, want = (None, None) if cases is None else cases[step - 1]
            st, nd, bodies, placed = ctx.reconcile_gangs(arena.pods(pods_s), 4, [0, 2, 4], [2, 2], json_cap=cap)
            assert st.tolist() == [0, 0, 0, 0] and nd.tolist() == [0, 0, -1, 0] and placed.tolist() == [2, 1]
            assert ctx.num_bound == 3  # the bodies that did not fit are still bound
            if cases is None:
                full, cases = bodies, string_list_cases(bodies)
                assert full[2] is None and all(b is not None for b in full[:2] + full[3:])
            else:
                assert bodies == want, cap
