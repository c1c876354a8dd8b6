"""Provisioning Solve latency while the deprovisioner sweeps, not part of bench.py. A C2- and a C4-shaped Solve (median of
7) in three setups: alone; while a C5-shaped single-node sweep (batch 64) runs on another context; and with that sweep
through the process-wide handle behind a caller-side mutex, the only safe way to share the library before contexts. The
sweep's own time is printed for each. One JSON line per Solve shape, with the card read in the same run."""
import argparse
import statistics
import threading
import time

from timing_lib import card, emit, load_pkg, need_device


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    cluster = pkg.Problem.synth(5, 50_000, 1000, 42, 5000)
    prov = pkg.Context(0)
    deprov = pkg.Context(0)
    lines = []
    for name, problem in (("C2", pkg.Problem.synth(2, 10_000, 500, 42, 0)), ("C4", pkg.Problem.synth(4, 100_000, 1000, 42, 0))):
        out = {"card": gpu, "solve": name, "sweep": "C5 single-node, batch 64", "reps": args.reps}
        for setup in ("alone", "with_context_sweep", "with_mutex_sweep"):
            mu = threading.Lock()
            sched = pkg.Scheduler(problem, context=None if setup == "with_mutex_sweep" else prov)
            session = None if setup == "alone" else pkg.ClusterSession(cluster, context=deprov if setup == "with_context_sweep" else None)

            def solve():
                if setup == "with_mutex_sweep":
                    with mu:
                        return sched.solve(count_visited=False)
                return sched.solve(count_visited=False)
            solve()
            stop = threading.Event()
            sweeps = []

            def sweep():
                n = session.n_candidates
                while not stop.is_set():
                    t0 = time.perf_counter()
                    for lo in range(0, n, 64):
                        if setup == "with_mutex_sweep":
                            with mu:
                                session.probe_sets([[i] for i in range(lo, min(n, lo + 64))], False)
                        else:
                            session.probe_sets([[i] for i in range(lo, min(n, lo + 64))], False)
                        if stop.is_set():
                            return
                    sweeps.append(time.perf_counter() - t0)
            th = threading.Thread(target=sweep) if session else None
            if th:
                th.start()
                time.sleep(0.5)
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                solve()
                ts.append(time.perf_counter() - t0)
            if th:
                while not sweeps:  # at least one whole sweep next to the Solves
                    time.sleep(0.05)
                stop.set()
                th.join()
                session.close()
            out[f"solve_ms_{setup}"] = 1000 * statistics.median(ts)
            if sweeps:
                out[f"sweep_ms_{setup}"] = 1000 * statistics.median(sweeps)
        lines.append(out)
    emit(lines, args.out)
    deprov.destroy()
    prov.destroy()


if __name__ == "__main__":
    main()
