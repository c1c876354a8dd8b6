"""Timing of a C4-shaped Solve (2 000 existing nodes, a batch of deployments) with and without a hostname NotIn [5 nodes]
requirement on its largest deployment, not part of bench.py. The requirement makes the deployment's class a table entry
(DESIGN.md §3, hostname requirements), which the existing-node run accepts, skipping the 5 excluded slots. Prints one JSON
line per variant: medians of --reps resident pack times and of end-to-end Solves, the pods placed on existing nodes (which
the generic step would place on the same nodes: whether the existing-node run took them is read off the pack time, not
counted), and the card name and power limit read in the same run.

    python tests/gpu_hostname_timing.py [--reps R] [--out FILE]
"""
import argparse
import random
import statistics

import fixtures as fx
from timing_lib import card, emit, load_pkg, need_device


def c4_dict(excluded, nodes=2000, deployments=20, types=400, seed=4):
    rng = random.Random(seed)
    its = fx.fake_instance_types(types)
    ns = []
    for i in range(nodes):
        it = its[rng.choice([3, 7, 15])]
        ns.append(fx.state_node(f"n{i:04d}", it["name"], zone=fx.ZONES[i % 3], allocatable=it["capacity"], capacity=it["capacity"]))
    pods = []
    for d in range(deployments):
        n = 12000 if d == 0 else rng.randint(300, 1500)
        kw = {"labels": {"app": f"d{d}"}}
        if d == 0 and excluded:
            kw["nodeAffinity"] = {"required": [[{"key": fx.HOSTNAME, "operator": "NotIn", "values": [f"n{i:04d}" for i in excluded]}]]}
        req = {"cpu": rng.choice(["250m", "500m", "1"]), "memory": rng.choice(["256Mi", "512Mi", "1Gi"])}
        pods += [fx.pod(dict(req), **kw) for _ in range(n)]
    rng.shuffle(pods)
    return fx.problem(pods, instance_types=its, nodes=ns)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    variants = {"plain": c4_dict(()), "notin5": c4_dict((0, 1, 2, 3, 4))}
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
                n_ex = len(d["existing"])
                big = [i for i, p in enumerate(variants[k]["pods"]) if p["labels"]["app"] == "d0"]
                lines.append({"card": gpu, "variant": k, "pods": len(variants[k]["pods"]), "existing_nodes": n_ex,
                              "pack_ms_median": statistics.median(pack[k]), "solve_ms_median": statistics.median(solve[k]),
                              "largest_deployment_on_existing": sum(1 for i in big if 0 <= d["assign"][i] < n_ex),
                              "largest_deployment_on_excluded": sum(1 for i in big if 0 <= d["assign"][i] < 5),
                              "hostname_words": rs.dims["hostname_words"]})
    emit(lines, a.out)


if __name__ == "__main__":
    main()
