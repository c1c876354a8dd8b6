"""K1 / K2 / end-to-end times of a C4-shaped batch (100 000 pods in deployments of 250, a quarter with hostname anti-affinity,
half with zone spread, a quarter with hostname spread) over an 800-type cloud catalog, with 16, 32 and 64 provisioners that
name template-only keys (tests/provisioner_problems.py). Prints one JSON line per provisioner count; F is the dense
pods x (template, type) feasibility matrix, P x V x W32 words of 4 bytes.

    python tests/gpu_provisioner_timing.py [--pods N] [--reps R] [--out FILE]
"""
import argparse
import random
import statistics
import time

import fixtures as fx
import provisioner_problems as pp
from timing_lib import emit, load_pkg, need_device

CPU = ["100m", "250m", "500m", "1", "1500m"]
MEM = ["100Mi", "256Mi", "512Mi", "1Gi", "2Gi", "4Gi"]


def c4_pods(n, rng):
    pods = []
    for d in range((n + 249) // 250):
        app = f"d{d}"
        spec = {"labels": {"app": app}}
        if rng.random() < 0.25:
            spec["podAntiAffinity"] = {"required": [fx.affinity_term(fx.HOSTNAME, {"app": app})]}
        ts = []
        if rng.random() < 0.5:
            ts.append(fx.spread(fx.ZONE, {"app": app}))
        if rng.random() < 0.25:
            ts.append(fx.spread(fx.HOSTNAME, {"app": app}, max_skew=rng.choice([1, 2, 4])))
        if ts:
            spec["topologySpreadConstraints"] = ts
        req = {"cpu": rng.choice(CPU), "memory": rng.choice(MEM)}
        pods += [fx.pod(dict(req), **spec) for _ in range(min(250, n - len(pods)))]
    return pods


def problem(n_pods, n_prov, seed=42):
    rng = random.Random(seed)
    its, families = pp.catalog(0, n=800)
    provs = pp.provisioners(n_prov, rng, families, [it["name"] for it in its])
    for pr in provs:
        pr.pop("limits", None)
        pr.pop("taints", None)
    return fx.problem(c4_pods(n_pods, rng), instance_types=its, provisioners=provs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    lines = []
    for v in (16, 32, 64):
        d = problem(a.pods, v)
        prob = pkg.Problem.from_dict(d)
        t0 = time.perf_counter()
        rs = pkg.ResidentSolve(prob)
        encode_ms = (time.perf_counter() - t0) * 1e3
        rs.set_count_visited(False)
        rs.load()
        k1c, k1, k2 = [], [], []
        for i in range(a.reps + 1):
            rs.run()
            res = rs.download()
            tm = rs.timings()
            if i:
                k1c.append(tm["class_feasibility_us"]); k1.append(tm["feasibility_us"]); k2.append(tm["pack_us"])
        e2e = []
        for i in range(a.reps + 1):
            us, _ = rs.solve_e2e()
            if i:
                e2e.append(us)
        dims = rs.dims
        f_bytes = dims["pods"] * dims["templates"] * dims["type_words"] * 8
        line = {"provisioners": v, "pods": dims["pods"], "types": dims["types"], "templates": dims["templates"], "mask_keys": dims["keys"],
                "folded": rs.key_info(pp.PROVISIONER_NAME) is None, "new_nodes": res.num_new_nodes,
                "k1_class_ms": statistics.median(k1c) / 1e3, "k1_ms": statistics.median(k1) / 1e3, "k2_ms": statistics.median(k2) / 1e3,
                "e2e_solve_ms": statistics.median(e2e) / 1e3, "encode_ms": encode_ms, "F_MB": f_bytes / 1e6}
        lines.append(line)
        del rs
    emit(lines, a.out)


if __name__ == "__main__":
    main()
