"""Time per candidate set of simulateScheduling's whole result on C5 (5 000 nodes, 50 000 bound pods, 1 000 instance types):
ClusterSession.simulate on the device-resident cluster, one set per call and 20 per call, against
Scheduler.solve(candidates=set), which encodes and uploads the whole cluster for every set. Single-node sets, as Expiration
and Drift pass them. Medians of 3 calls after a warm-up; the card's name, power limit and maximum SM clock go beside them.

    python tests/gpu_full_sim_timing.py [--out FILE]
"""
import argparse

import timing_lib as tl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    pkg = tl.load_pkg()
    tl.need_device(pkg)
    problem = pkg.Problem.synth(5, 50000, 1000, 42, 5000)
    cs = pkg.ClusterSession(problem)
    assert cs.resident
    nodes = cs.candidate_nodes()[:20]
    one_ms, got = tl.timed(lambda: cs.simulate([nodes[:1]])[0], args.reps)
    batch_ms, _ = tl.timed(lambda: cs.simulate([[n] for n in nodes]), args.reps)
    solve_ms, want = tl.timed(lambda: pkg.Scheduler(problem).solve(candidates=nodes[:1], count_visited=False), args.reps)
    same = got.to_dict(True)["assign"] == want.to_dict(True)["assign"] and got.to_dict(True)["newNodes"] == want.to_dict(True)["newNodes"]
    tl.emit([{"workload": "C5 single-node sets", "card": tl.card(), "reps": args.reps, "same_result": same,
              "simulate_1_per_call_ms_per_set": round(one_ms, 3), "simulate_20_per_call_ms_per_set": round(batch_ms / len(nodes), 3),
              "solve_ms_per_set": round(solve_ms, 3)}], args.out)


if __name__ == "__main__":
    main()
