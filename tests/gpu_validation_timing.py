"""Timing of consolidation validation on a C5-shaped cluster (5 000 nodes, 50 000 bound pods, 1 000 instance types), not part
of bench.py. Two clusters after the TTL: unchanged (every command validates) and saturated by pending pods that fit
nowhere (nothing validates, so the single-node sweep validates every actionable candidate). Prints one JSON line with the
card name and power limit read in the same run."""
import argparse
import time

import fixtures as fx
from timing_lib import card, emit, load_pkg, need_device, sweep_singles, timed


def c5_dict(nodes=5000, pods_per_node=10, types=1000):
    its = fx.fake_instance_types(types)
    big = its[-1]
    ns = []
    for i in range(nodes):
        pods_ = [fx.pod({"cpu": "100m", "memory": "128Mi"}, nodeName=f"n{i}", labels={"app": f"a{j % 50}"}) for j in range(pods_per_node)]
        ns.append(fx.state_node(f"n{i}", big["name"], zone=fx.ZONES[i % 3], allocatable=big["capacity"], pods_=pods_))
    return fx.problem([], instance_types=its, provisioners=[fx.provisioner(consolidationEnabled=True, limits=None)], nodes=ns, deriveCandidates=True)


def main():
    argparse.ArgumentParser().parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    b = c5_dict()
    before = pkg.Problem.from_dict(b)
    unchanged = pkg.Problem.from_dict(b)
    b["pods"] = [fx.pod({"cpu": "100000"}) for _ in range(4)]
    saturated = pkg.Problem.from_dict(b)
    out = {"card": gpu, "nodes": 5000, "bound_pods": 50000, "instance_types": 1000}
    cs = pkg.ClusterSession(before)
    cmd = [([0], *cs.probe_sets([[0]], False)[0])]
    t0 = time.perf_counter()
    cs.validate(unchanged, cmd)
    out["open_validation_snapshot_ms"] = 1000 * (time.perf_counter() - t0)
    cs.close()
    multi = pkg.MultiNodeConsolidation(before)
    out["multi_node_no_validation_ms"], r0 = timed(multi.first_n_node_consolidation_option, 3)
    out["multi_node_validated_unchanged_ms"], r1 = timed(lambda: multi.compute_command(unchanged), 3)
    out["multi_node_validated_saturated_ms"], r2 = timed(lambda: multi.compute_command(saturated), 3)
    out["multi_node_actions"] = [r0["action"], r1["action"], r2["action"]]
    single = pkg.SingleNodeConsolidation(before)
    out["single_node_all_candidates_no_validation_ms"], _ = timed(lambda: sweep_singles(pkg, before), 1)
    out["single_node_validated_saturated_ms"], r3 = timed(lambda: single.compute_command(batch=64, after=saturated), 1)
    out["single_node_saturated_validations"] = len(r3["validations"])
    out["single_node_saturated_action"] = r3["action"]
    emit([out], None)


if __name__ == "__main__":
    main()
