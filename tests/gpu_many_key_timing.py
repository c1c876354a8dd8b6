"""Timing of a C4-shaped batch (100 000 pods in 20 deployments) on the cloud-shaped catalog of tests/many_key_problems.py
(800 instance types with requirements on 12 keys), not part of bench.py. Variant `12keys`: every deployment names 12 label keys
through its node selector and required term, half of them with a zone spread (DESIGN.md §3, touched keys); the pack kernel
refused such classes before, so that variant has no earlier figure. Variant `6keys`: the same batch with each deployment cut
to its first 6 keys. Prints one JSON line per variant: medians of --reps resident K1 (feasibility) and K2 (pack) times and of
end-to-end Solves, the pods placed, and the card name and power limit read in the same run.

    python tests/gpu_many_key_timing.py [--reps R] [--out FILE]
"""
import argparse
import random
import statistics

import fixtures as fx
import many_key_problems as mk
from timing_lib import card, emit, load_pkg, need_device


def c4_dict(n_keys, pods=100_000, deployments=20, seed=4):
    rng = random.Random(seed)
    its, families = mk.types(seed)
    fams = mk._x86(families)
    out = []
    for d in range(deployments):
        app = f"d{d}"
        team = "ml" if d % 2 else "web"
        reqs = [mk._r(fx.ARCH, "In", "amd64"), mk._r(fx.OS, "In", "linux"), mk._r("team", "In", team), mk._r("env", "In", "prod"),
                mk._r("category", "In", "c", "m", "r"), mk._r("generation", "Gt", 3), mk._r(fx.CAPACITY_TYPE, "In", "spot", "on-demand"),
                mk._r("family", "NotIn", *rng.sample(fams, 4)), mk._r("cpu", "Gt", 1), mk._r("memory", "Lt", 262144),
                mk._r("size", "NotIn", "medium"), mk._r("nvme", "Exists")][:n_keys]
        kw = {"labels": {"app": app}, "nodeAffinity": {"required": [reqs]}}
        if d % 2 == 0:
            kw["topologySpreadConstraints"] = [fx.spread(fx.ZONE, {"app": app})]
        req = {"cpu": rng.choice(["100m", "250m", "500m"]), "memory": rng.choice(["128Mi", "256Mi", "512Mi"])}
        n = pods // deployments
        out += [fx.pod(dict(req), name=f"{app}-{i:05d}", uid=f"{app}-{i:05d}", creationTimestamp=d, **kw) for i in range(n)]
    return fx.problem(out, instance_types=its, provisioners=mk.provisioners(limits=False), wellKnownLabels=mk.WELL_KNOWN)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    variants = {"12keys": 12, "6keys": 6}
    problems = {k: pkg.Problem.from_dict(c4_dict(n)) for k, n in variants.items()}
    k1 = {k: [] for k in variants}
    k2 = {k: [] for k in variants}
    solve = {k: [] for k in variants}
    lines = []
    for rep in range(a.reps + 1):  # alternating; the first round warms every variant up
        for k, problem in problems.items():
            rs = pkg.ResidentSolve(problem)
            rs.set_count_visited(False)
            rs.load()
            rs.run()
            t = rs.timings()
            res, ph = pkg.solve_timed(problem)
            if rep:
                k1[k].append(t["feasibility_us"] / 1000)
                k2[k].append(t["pack_us"] / 1000)
                solve[k].append(ph["total_us"] / 1000)
            if rep == a.reps:
                d = res.to_dict()
                lines.append({"card": gpu, "variant": k, "pods": rs.dims["pods"], "types": rs.dims["types"], "keys": rs.dims["keys"],
                              "k1_ms_median": statistics.median(k1[k]), "k2_ms_median": statistics.median(k2[k]),
                              "solve_ms_median": statistics.median(solve[k]),
                              "placed": sum(1 for x in d["assign"] if x >= 0), "new_nodes": len(d["newNodes"])})
    emit(lines, a.out)


if __name__ == "__main__":
    main()
