"""Timing of consolidation on a C5-shaped cluster (5 000 nodes, 50 000 bound pods, 1 000 instance types) whose pods mount
volume claims, not part of bench.py. About a third of the bound pods are StatefulSet pods with an EBS claim of their own
(every node limits EBS to 25), and --deploy deployments have two replicas on different nodes that share one claim, so more
than 64 claims are tracked and the claim table exists. Before the claim table this cluster was refused, so it has no
"before" figure. Run twice: with the claims and with every claim stripped. Times the multi-node search and the single-node
sweep over every candidate, medians of --reps. Then a Solve batch of deployments whose replicas share --claims claims on
2 000 existing nodes: pack kernel and end to end, medians of --reps. One JSON line per run, with the card name and power
limit read in the same run.

    python tests/gpu_volume_timing.py [--reps R] [--deploy N] [--claims N] [--out FILE]
"""
import argparse
import statistics

import fixtures as fx
from timing_lib import card, emit, load_pkg, need_device, sweep_singles, timed
import volume_problems as vp


def c5_dict(claims, deploy, nodes=5000, pods_per_node=10, types=1000):
    its = fx.fake_instance_types(types)
    big = its[-1]
    provs = [fx.provisioner("default", consolidationEnabled=True, limits=None)]
    ns = []
    for i in range(nodes):
        name = f"n{i}"
        pods_ = [fx.pod({"cpu": "100m", "memory": "128Mi"}, nodeName=name, labels={"app": f"a{j % 50}"}) for j in range(pods_per_node - 3)]
        for k in range(3):  # StatefulSet pods, one claim each (one slot of the three is a deployment replica below)
            vs = [vp.vol(vp.EBS, f"db/data-{i}-{k}")] if claims else []
            pods_.append(fx.pod({"cpu": "250m", "memory": "256Mi"}, nodeName=name, labels={"app": "db"}, volumes=vs))
        ns.append(fx.state_node(name, big["name"], zone=fx.ZONES[i % 3], allocatable=big["capacity"], pods_=pods_,
                                volumeLimits={vp.EBS: 25}))
    for d in range(deploy if claims else 0):  # replicas on nodes d and d + nodes/2 share a claim
        for i in (d, d + nodes // 2):
            p = ns[i]["pods"][-1]
            p["labels"] = {"app": f"web-{d}"}
            p["volumes"] = [vp.vol(vp.EBS, f"web/cache-{d}")]
    return fx.problem([], instance_types=its, provisioners=provs, nodes=ns, deriveCandidates=True)


def solve_dict(claims, nodes=2000, types=1000):
    its = fx.fake_instance_types(types)
    big = its[-1]
    ns = [fx.state_node(f"e{i}", big["name"], zone=fx.ZONES[i % 3], allocatable=big["capacity"], volumeLimits={vp.EBS: 8},
                        pods_=[fx.pod({"cpu": "100m", "memory": "128Mi"}, nodeName=f"e{i}", volumes=[vp.vol(vp.EBS, f"db/own-{i}-{k}")])
                               for k in range(4)])
          for i in range(nodes)]
    pods = []
    for d in range(claims):
        pods += [fx.pod({"cpu": "250m", "memory": "256Mi"}, labels={"app": f"dep-{d}"}, volumes=[vp.vol(vp.EBS, f"app/claim-{d}")])
                 for _ in range(3)]
    pods += [fx.pod({"cpu": "250m", "memory": "256Mi"}, labels={"app": "sts"}, volumes=[vp.vol(vp.EBS, f"sts/new-{i}")]) for i in range(2000)]
    return fx.problem(pods, instance_types=its, nodes=ns)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--deploy", type=int, default=200)
    ap.add_argument("--claims", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    lines = []
    for claims in (True, False):
        d = c5_dict(claims, a.deploy)
        problem = pkg.Problem.from_dict(d)
        line = {"card": gpu, "workload": "cluster", "nodes": len(d["nodes"]), "bound_pods": sum(len(n["pods"]) for n in d["nodes"]),
                "claims": sum(len(p.get("volumes", [])) for n in d["nodes"] for p in n["pods"])}
        multi = pkg.MultiNodeConsolidation(problem)
        line["multi_node_search_ms"], r = timed(multi.first_n_node_consolidation_option, a.reps)
        line["multi_node_action"], line["multi_node_removed"] = r["action"], r["nodes_removed"]

        line["single_node_sweep_ms"], acts = timed(lambda: sweep_singles(pkg, problem), a.reps)
        line["single_node_candidates"] = len(acts)
        line["single_node_actionable"] = sum(1 for x in acts if x in (1, 2))
        lines.append(line)
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(solve_dict(a.claims)))
    rs.set_count_visited(False)
    rs.load()
    k2, tot = [], []
    for i in range(a.reps + 1):
        rs.run()
        t = rs.timings()
        if i:
            k2.append(t["pack_us"]); tot.append(t["total_us"])
    e2e = statistics.median(rs.solve_e2e()[0] for _ in range(a.reps))
    line = {"card": gpu, "workload": "solve", "existing": rs.dims["existing"], "pods": rs.dims["pods"], "classes": rs.dims["classes"],
            "volume_claims": rs.dims["volume_claims"], "volume_ext_words": rs.dims["volume_ext_words"],
            "k2_ms": statistics.median(k2) / 1000, "resident_ms": statistics.median(tot) / 1000, "e2e_ms": e2e / 1000}
    lines.append(line)
    emit(lines, a.out)


if __name__ == "__main__":
    main()
