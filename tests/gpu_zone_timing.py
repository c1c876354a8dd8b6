"""Timing of a C4-shaped batch (100 000 pods in 20 deployments, 1 000 instance types) on a 3-zone catalog and on a 20-zone
catalog (6 AZs and 14 Local Zones, DESIGN.md §3, offering slots), not part of bench.py. The 20-zone runs spread their
zone-spread deployments once over the AZs a provisioner allows and once over all zones. Prints one JSON line per variant:
medians of --reps resident K1 (feasibility) and K2 (pack) times and of end-to-end Solves, the offering slots of the
encoding, the pods placed, and the card name and power limit read in the same run.

    python tests/gpu_zone_timing.py [--reps R] [--out FILE]
"""
import argparse
import random
import statistics

import fixtures as fx
from timing_lib import card, emit, load_pkg, need_device
from zone_problems import AZS, local_zones


def catalog(zones, local, types=1000):
    """`types` instance types offered spot and on-demand in `zones`; the 50 smallest also on-demand in `local`"""
    its = []
    for i in range(types):
        res = {"cpu": str(1 + i % 64), "memory": f"{2 + (i * 7) % 256}Gi", "pods": "110"}
        price = fx.price_from_resources(res) + i * 1e-4
        offers = [{"capacityType": ct, "zone": z, "price": round(price * (0.6 if ct == "spot" else 1.0), 6), "available": True}
                  for z in zones for ct in ("spot", "on-demand")]
        if i < 50:
            offers += [{"capacityType": "on-demand", "zone": z, "price": round(price * 1.2, 6), "available": True} for z in local]
        its.append(fx.instance_type(f"t{i:04d}", res, offerings=offers, oses=("linux",)))
    return its


def c4_dict(variant, pods=100_000, deployments=20, seed=4):
    rng = random.Random(seed)
    local = [] if variant == "3zones" else local_zones(14)
    zones = fx.ZONES if variant == "3zones" else AZS
    its = catalog(zones, local)
    if variant == "20zones-azs":
        # the spreads' domains are the 6 AZs the provisioner allows; the Local Zones stay dictionary values (offerings name them)
        provs = [{"name": "azs", "requirements": [{"key": fx.ZONE, "operator": "In", "values": AZS}]}]
    else:
        provs = [{"name": "default", "requirements": [{"key": fx.ZONE, "operator": "In", "values": list(zones) + local}]}]
    out = []
    for d in range(deployments):
        n = pods // deployments
        app = f"d{d}"
        kw = {"labels": {"app": app}}
        if d % 2 == 0:
            kw["topologySpreadConstraints"] = [fx.spread(fx.ZONE, {"app": app})]
        req = {"cpu": rng.choice(["100m", "250m", "500m"]), "memory": rng.choice(["128Mi", "256Mi", "512Mi"])}
        out += [fx.pod(dict(req), name=f"{app}-{i:05d}", uid=f"{app}-{i:05d}", creationTimestamp=d, **kw) for i in range(n)]
    return fx.problem(out, instance_types=its, provisioners=provs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    variants = ("3zones", "20zones-azs", "20zones-all")
    problems = {k: pkg.Problem.from_dict(c4_dict(k)) for k in variants}
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
                lines.append({"card": gpu, "variant": k, "pods": rs.dims["pods"], "types": rs.dims["types"],
                              "offering_slots": rs.dims["offering_slots"], "k1_ms_median": statistics.median(k1[k]),
                              "k2_ms_median": statistics.median(k2[k]), "solve_ms_median": statistics.median(solve[k]),
                              "placed": sum(1 for x in d["assign"] if x >= 0), "new_nodes": len(d["newNodes"])})
    emit(lines, a.out)


if __name__ == "__main__":
    main()
