"""What the GPU timing scripts (tests/gpu_*_timing.py) share: the import path, the device check, the card line recorded
beside every figure, the median timer, the single-node sweep and the JSON-lines output. Not collected by pytest."""
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from conftest import load_pkg  # noqa: E402,F401


def need_device(pkg):
    if pkg.device_count() < 1:
        raise SystemExit("needs a CUDA device")


def card():
    """name, power limit and maximum SM clock of the card, read in the same run as the figures"""
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def timed(fn, reps):
    """one warm-up call, then the median of `reps` calls in ms, and the last call's output"""
    fn()
    ts, out = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return 1000 * statistics.median(ts), out


def sweep_singles(pkg, problem, batch=64):
    """single-node consolidation of every candidate, `batch` simulations per call, on a fresh session -> each action"""
    s = pkg.ClusterSession(problem)
    acts = []
    for lo in range(0, s.n_candidates, batch):
        acts += [x[0] for x in s.probe_sets([[i] for i in range(lo, min(s.n_candidates, lo + batch))], False)]
    s.close()
    return acts


def emit(lines, out):
    """print each result as one JSON line and, when `out` is given, write them all there"""
    for x in lines:
        print(json.dumps(x), flush=True)
    if out:
        Path(out).parent.mkdir(parents=True, exist_ok=True)
        Path(out).write_text("\n".join(json.dumps(x) for x in lines) + "\n")
