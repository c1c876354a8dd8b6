"""Timing of a C4-shaped Solve (2 000 existing nodes, a batch of deployments) in which a share of the deployments is pinned to
instance-type lists and spread over zones, not part of bench.py. Variant "itype" pins through node.kubernetes.io/instance-type,
so the spreads' node filters name the key and the problem gets the instance-type filter tables (DESIGN.md §3, instance-type
node filters); variant "label" pins the same deployments to the same types through the `integer` label those types carry,
which needs no table. Prints one JSON line per variant: medians of --reps resident pack times and of end-to-end Solves, the
pods placed, and the card name and power limit read in the same run.

    python tests/gpu_itype_filter_timing.py [--reps R] [--out FILE]
"""
import argparse
import random
import statistics

import fixtures as fx
from timing_lib import card, emit, load_pkg, need_device


def c4_dict(via_itype, nodes=2000, deployments=20, pinned=6, types=400, seed=4):
    rng = random.Random(seed)
    its = fx.fake_instance_types(types)
    ns = []
    for i in range(nodes):
        it = its[rng.choice([3, 7, 15])]
        ns.append(fx.state_node(f"n{i:04d}", it["name"], zone=fx.ZONES[i % 3], allocatable=it["capacity"], capacity=it["capacity"]))
    pods = []
    for d in range(deployments):
        n = 8000 if d == 0 else rng.randint(300, 1500)
        lab = {"app": f"d{d}"}
        kw = {"labels": lab}
        if d < pinned:
            listed = sorted(rng.sample(range(types), 6) + [7])
            if via_itype:
                req = {"key": fx.INSTANCE_TYPE, "operator": "In", "values": [its[i]["name"] for i in listed]}
            else:  # fake-it-i carries integer = i + 1 (fixtures.instance_type), a value no other type has
                req = {"key": "integer", "operator": "In", "values": [str(i + 1) for i in listed]}
            kw["nodeAffinity"] = {"required": [[req]]}
            kw["topologySpreadConstraints"] = [fx.spread(fx.ZONE, lab, max_skew=1)]
        r = {"cpu": rng.choice(["250m", "500m", "1"]), "memory": rng.choice(["256Mi", "512Mi", "1Gi"])}
        pods += [fx.pod(dict(r), **kw) for _ in range(n)]
    rng.shuffle(pods)
    return fx.problem(pods, instance_types=its, nodes=ns)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    variants = {"label": c4_dict(False), "itype": c4_dict(True)}
    problems = {k: pkg.Problem.from_dict(v) for k, v in variants.items()}
    pack = {k: [] for k in variants}
    solve = {k: [] for k in variants}
    lines = []
    for rep in range(a.reps + 1):  # alternating; the first round warms both up
        for k, problem in problems.items():
            rs = pkg.ResidentSolve(problem)
            rs.set_count_visited(False)
            rs.load()
            rs.run()
            t = rs.timings()["pack_us"]
            res, ph = pkg.solve_timed(problem)
            if rep:
                pack[k].append(t / 1000)
                solve[k].append(ph["total_us"] / 1000)
            if rep == a.reps:
                d = res.to_dict()
                lines.append({"card": gpu, "variant": k, "pods": len(variants[k]["pods"]),
                              "pack_ms_median": statistics.median(pack[k]), "solve_ms_median": statistics.median(solve[k]),
                              "placed": sum(1 for x in d["assign"] if x >= 0), "itype_filter_terms": rs.dims["itype_filter_terms"]})
    emit(lines, a.out)


if __name__ == "__main__":
    main()
