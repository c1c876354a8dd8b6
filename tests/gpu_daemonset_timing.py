"""Timing of problems whose daemonsets select nodes by instance type (DESIGN.md §3, daemonset overhead), not part of
bench.py. Before the encoder charged such daemonsets, every one of these problems was refused, so there is no "before"
figure to compare with.

 * c4: a C4-shaped batch (2 000 existing nodes, 20 deployments, about 21 000 pods) on the mixed catalog of
   tests/daemonset_itype_problems.py with three plugin daemonsets (Neuron, EFA, a monitor kept off small types): medians of
   --reps encodes, K1 (feasibility) and K2 (pack) kernel times of a resident solve, and end-to-end Solves;
 * c5: a C5-shaped cluster (2 000 nodes with bound web and plugin pods, 1 000 candidates): cluster load (session creation),
   the multi-node binary search and a 512-candidate single-node sweep, medians of --reps.

Prints one JSON line per workload with the card name and power limit read in the same run.

    python tests/gpu_daemonset_timing.py [--reps R] [--out FILE]
"""
import argparse
import copy
import random
import statistics
import time

import daemonset_itype_problems as dp
import fixtures as fx
from timing_lib import card, emit, load_pkg, need_device

GENERAL = ["m5.large", "m5.xlarge", "m5.2xlarge", "c5.xlarge", "c5.4xlarge"]


def _plugins():
    neuron, efa = dp._cluster_daemons()
    monitor = dp._daemon("250m", "256Mi", nodeAffinity={"required": [[dp._it("NotIn", dp.SMALL_TYPES)]]})
    return [neuron, efa, monitor]


def _nodes(rng, n, web):
    out = []
    types = GENERAL + dp.NEURON_TYPES[:3] + ["p4d.24xlarge"]
    daemons = _plugins()
    for i in range(n):
        x, t = f"n{i:04d}", types[rng.randrange(len(types))]
        cpu = min(int(next(it for it in dp.TYPES if it["name"] == t)["capacity"]["cpu"]), 16)
        bound = [fx.pod({"cpu": rng.choice(["300m", "700m", "1"]), "memory": "512Mi"}, nodeName=x, labels={"app": "web"})
                 for _ in range(rng.randint(0, web))]
        for d, sel in zip(daemons, (dp.NEURON_TYPES, dp.EFA_TYPES, None)):
            if sel is None or t in sel:
                bound.append(dict(copy.deepcopy(d), nodeName=x, isDaemonSet=True, name=f"ds-{x}-{len(bound)}", uid=f"uid-ds-{x}-{len(bound)}"))
        out.append(dp._node(x, t, rng, cpu=cpu, pods=bound))
    return out


def c4_dict(nodes=2000, deployments=20, seed=4):
    rng = random.Random(seed)
    prov = [fx.provisioner("neuron", weight=10, taints=[dp.NEURON_TAINT], requirements=[dp._it("In", dp.NEURON_TYPES)],
                           limits={"cpu": "100000"}),
            fx.provisioner("default", limits={"cpu": "100000"})]
    pods = []
    for d in range(deployments):
        n = 8000 if d == 0 else rng.randint(300, 1000)
        r = {"cpu": rng.choice(["250m", "500m", "1"]), "memory": rng.choice(["256Mi", "512Mi", "1Gi"])}
        kw = {"labels": {"app": f"d{d}"}}
        if d % 5 == 1:
            r[dp.NEURON] = "1"
            kw.update(tolerations=dp.NEURON_TOL, nodeSelector={fx.PROVISIONER_NAME: "neuron"})
        pods += [fx.pod(dict(r), **kw) for _ in range(n)]
    rng.shuffle(pods)
    return dp._problem(pods, _plugins(), _nodes(rng, nodes, 3), provisioners=prov)


def c5_dict(nodes=2000, candidates=1000, seed=5):
    rng = random.Random(seed)
    ns = _nodes(rng, nodes, 6)
    for k in range(candidates):
        ns[k].update(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(k))
    return dp._problem([], _plugins(), ns, provisioners=[fx.provisioner("default", limits={"cpu": "100000"})])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    lines = []

    c4 = c4_dict()
    problem = pkg.Problem.from_dict(c4)
    enc, k1, k2, solve = [], [], [], []
    placed = None
    for rep in range(a.reps + 1):  # the first round warms up
        rs = pkg.ResidentSolve(problem)
        rs.set_count_visited(False)
        rs.load()
        rs.run()
        t = rs.timings()
        res, ph = pkg.solve_timed(problem)
        if rep:
            k1.append(t["feasibility_us"] / 1000)
            k2.append(t["pack_us"] / 1000)
            enc.append(ph["encode_us"] / 1000)
            solve.append(ph["total_us"] / 1000)
            placed = sum(1 for x in res.to_dict(brief=True)["assign"] if x >= 0)
    lines.append({"card": gpu, "workload": "c4-daemonsets", "pods": len(c4["pods"]), "existing": rs.dims["existing"],
                  "templates": rs.dims["templates"], "reps": a.reps, "encode_ms_median": statistics.median(enc),
                  "k1_ms_median": statistics.median(k1), "k2_ms_median": statistics.median(k2),
                  "solve_ms_median": statistics.median(solve), "placed": placed})

    c5 = pkg.Problem.from_dict(c5_dict())
    load, search, sweep = [], [], []
    for rep in range(a.reps + 1):
        t0 = time.perf_counter()
        mnc = pkg.MultiNodeConsolidation(c5)
        cs = mnc.session()
        t1 = time.perf_counter()
        full = mnc.first_n_node_consolidation_option()
        t2 = time.perf_counter()
        sw = cs.probe_sets([[i] for i in range(min(512, cs.n_candidates))], False)
        t3 = time.perf_counter()
        cs.close()
        if rep:
            load.append((t1 - t0) * 1000)
            search.append((t2 - t1) * 1000)
            sweep.append((t3 - t2) * 1000)
    lines.append({"card": gpu, "workload": "c5-daemonsets", "nodes": 2000, "candidates": cs.n_candidates, "reps": a.reps,
                  "cluster_load_ms_median": statistics.median(load), "multi_node_search_ms_median": statistics.median(search),
                  "single_node_sweep_512_ms_median": statistics.median(sweep), "action": full["action"],
                  "nodes_removed": full["nodes_removed"], "probes": len(full["probes"]), "sweep_hits": sum(1 for x, _ in sw if x)})
    emit(lines, a.out)


if __name__ == "__main__":
    main()
