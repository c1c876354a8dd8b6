"""Timing of consolidation on a C5-shaped cluster (5 000 nodes, 50 000 bound pods) of 64 dedicated pools, not part of bench.py.
Run twice: with a few hundred node-only taint sets (device taints of their own, cordoned nodes; taint-set ids of 64 and above,
read from the per-class table) and with those extra taints removed (every node carries exactly its pool's taint: 64 sets).
Times the multi-node search and the single-node sweep over every candidate, medians of --reps, and prints one JSON line per
run with the card name and power limit read in the same run.

    python tests/gpu_taintset_timing.py [--reps R] [--extra N] [--out FILE]
"""
import argparse

import fixtures as fx
import taint_problems as tp
from timing_lib import card, emit, load_pkg, need_device, sweep_singles, timed


def c5_dict(extra, nodes=5000, pods_per_node=10, types=1000, pools=64):
    """node i belongs to pool i % 64; the first `extra` nodes get a taint set no template has (a device taint of their own,
    every fourth one also cordoned). Bound pods tolerate either everything or every `dedicated` taint, so both kinds of
    node stay destinations."""
    its = fx.fake_instance_types(types)
    big = its[-1]
    provs = [fx.provisioner(f"pool-{i:02d}", consolidationEnabled=True, limits=None, taints=[tp.pool_taint(i)]) for i in range(pools)]
    everything, dedicated = [{"operator": "Exists"}], [{"key": "dedicated", "operator": "Exists"}]
    ns = []
    for i in range(nodes):
        taints = [tp.pool_taint(i % pools)]
        if i < extra:
            taints.append({"key": "example.com/device", "value": f"d{i}", "effect": "NoSchedule"})
            if i % 4 == 0:
                taints.append(tp.CORDON)
        pods_ = [fx.pod({"cpu": "100m", "memory": "128Mi"}, nodeName=f"n{i}", labels={"app": f"a{j % 50}"},
                        tolerations=everything if j % 2 else dedicated) for j in range(pods_per_node)]
        ns.append(fx.state_node(f"n{i}", big["name"], zone=fx.ZONES[i % 3], allocatable=big["capacity"], pods_=pods_,
                                provisioner_name=f"pool-{i % pools:02d}", taints=taints))
    return fx.problem([], instance_types=its, provisioners=provs, nodes=ns, deriveCandidates=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--extra", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    lines = []
    for extra in (a.extra, 0):
        d = c5_dict(extra)
        problem = pkg.Problem.from_dict(d)
        line = {"card": gpu, "nodes": len(d["nodes"]), "bound_pods": sum(len(n["pods"]) for n in d["nodes"]), "node_only_extra": extra,
                "taint_sets": len(tp.distinct_sets(d))}
        multi = pkg.MultiNodeConsolidation(problem)
        line["multi_node_search_ms"], r = timed(multi.first_n_node_consolidation_option, a.reps)
        line["multi_node_action"], line["multi_node_removed"] = r["action"], r["nodes_removed"]

        line["single_node_sweep_ms"], acts = timed(lambda: sweep_singles(pkg, problem), a.reps)
        line["single_node_candidates"] = len(acts)
        line["single_node_actionable"] = sum(1 for x in acts if x in (1, 2))
        lines.append(line)
    emit(lines, a.out)


if __name__ == "__main__":
    main()
