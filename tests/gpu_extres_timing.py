"""Timing of batches whose pods request ext resources (DESIGN.md §3, more than 8 resources), not part of bench.py.

 * batch: a C4-shaped batch (100 000 pods in deployments of 100, zone spread, hostname anti-affinity, hostname spread,
   1 000 instance types, no existing nodes) in which 0 %, 5 % and 30 % of the deployments also request ext resources
   (six resources every instance type offers, three of them per deployment). Limits on five quota resources fill the row
   slots, so all six are ext resources; the 0 % batch has no ext resource and gives the cost of the shape itself. Reports K1
   (class rows + matrix), K2, the resident total and end to end, medians of --reps, and how many pods request an ext
   resource (every one of them takes the generic step).
 * cluster: a C5-shaped GPU cluster (5 000 nodes, 50 000 bound pods), with and without ext requests on the bound pods;
   times the multi-node search and the single-node sweep over every candidate.

Prints one JSON line per run with the card name, power limit and clock read in the same run.

    python tests/gpu_extres_timing.py [--reps R] [--pods N] [--out FILE]
"""
import argparse
import statistics

import fixtures as fx
from timing_lib import card, emit, load_pkg, need_device, sweep_singles, timed

EXT = [f"example.com/accel-{i}" for i in range(6)]
QUOTA = {f"example.com/quota-{i}": "100000000" for i in range(5)}  # with cpu, memory, pods: the 8 row slots


def _types(n):
    its = fx.fake_instance_types(n)
    for i, it in enumerate(its):
        for k, r in enumerate(EXT):
            it["capacity"][r] = str(1 + (i + k) % 8)
    return its


def batch_dict(pods, ext_share):
    """deployments of 100 pods; every third has a zone spread, every third a hostname anti-affinity, every third a hostname
    spread; deployment d requests ext resources when d * ext_share falls on a new integer (evenly spread)"""
    out = []
    n_dep = pods // 100
    ext_deps = 0
    for d in range(n_dep):
        req = {"cpu": f"{100 + 10 * (d % 37)}m", "memory": f"{128 + 32 * (d % 11)}Mi"}
        ext = int((d + 1) * ext_share) > int(d * ext_share)
        if ext:
            ext_deps += 1
            for k in range(3):
                req[EXT[(d + 2 * k) % len(EXT)]] = "1"
        kw = {"labels": {"app": f"d{d}"}}
        if d % 3 == 0:
            kw["topologySpreadConstraints"] = [fx.spread(fx.ZONE, {"app": f"d{d}"})]
        elif d % 3 == 1:
            kw["podAntiAffinity"] = {"required": [fx.affinity_term(fx.HOSTNAME, {"app": f"d{d}"})]}
        else:
            kw["topologySpreadConstraints"] = [fx.spread(fx.HOSTNAME, {"app": f"d{d}"}, max_skew=5)]
        out += [fx.pod(dict(req), **kw) for _ in range(100)]
    return fx.problem(out, instance_types=_types(1000), provisioners=[fx.provisioner(limits=QUOTA)]), ext_deps * 100


def cluster_dict(ext, nodes=5000, pods_per_node=10, types=1000):
    its = _types(types)
    big = its[-1]
    ns = []
    for i in range(nodes):
        ps = []
        for j in range(pods_per_node):
            req = {"cpu": "100m", "memory": "128Mi"}
            if ext and j % 3 == 0:
                req[EXT[(i + j) % len(EXT)]] = "1"
            ps.append(fx.pod(req, nodeName=f"n{i}", labels={"app": f"a{j % 50}"}))
        ns.append(fx.state_node(f"n{i}", big["name"], zone=fx.ZONES[i % 3], allocatable=big["capacity"], pods_=ps))
    return fx.problem([], instance_types=its, provisioners=[fx.provisioner(consolidationEnabled=True, limits=QUOTA)], nodes=ns,
                      deriveCandidates=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pods", type=int, default=100_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    lines = []
    for share in (0.0, 0.05, 0.30):
        d, ext_pods = batch_dict(a.pods, share)
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(d))
        rs.set_count_visited(False)
        rs.load()
        k1, k2, tot = [], [], []
        for i in range(a.reps + 1):
            rs.run()
            t = rs.timings()
            if i:
                k1.append(t["feasibility_us"]); k2.append(t["pack_us"]); tot.append(t["total_us"])
        e2e = statistics.median(rs.solve_e2e()[0] for _ in range(a.reps))
        line = {"card": gpu, "workload": "batch", "pods": a.pods, "ext_share": share, "ext_pods_generic_step": ext_pods,
                "resources": rs.dims["resources"], "resources_ext": rs.dims["resources_ext"], "classes": rs.dims["classes"],
                "k1_ms": statistics.median(k1) / 1000, "k2_ms": statistics.median(k2) / 1000, "resident_ms": statistics.median(tot) / 1000,
                "e2e_ms": e2e / 1000}
        lines.append(line)
    for ext in (True, False):
        problem = pkg.Problem.from_dict(cluster_dict(ext))
        line = {"card": gpu, "workload": "cluster", "nodes": 5000, "bound_pods": 50000, "ext_requests": ext}
        multi = pkg.MultiNodeConsolidation(problem)
        line["multi_node_search_ms"], r = timed(multi.first_n_node_consolidation_option, a.reps)
        line["multi_node_action"], line["multi_node_removed"] = r["action"], r["nodes_removed"]

        line["single_node_sweep_ms"], acts = timed(lambda: sweep_singles(pkg, problem), a.reps)
        line["single_node_candidates"] = len(acts)
        lines.append(line)
    emit(lines, a.out)


if __name__ == "__main__":
    main()
