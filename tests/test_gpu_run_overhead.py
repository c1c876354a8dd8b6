"""GPU: the class run's fixed path around its loop - per-node inputs, write-back and the compaction of the active list -
under both pack_kernel instantiations (blocks of up to 256 threads launch the one with the larger register budget, larger
blocks the other). Compared with the oracle at 32, 128, 256 and 512 threads: seeded problems whose class runs fill nodes
up to their pod capacity, so runs end with closed nodes (tombstones) at the front, in the middle and at the back of the
active list; and the full-size C2 / C3 / C4 results at 512 threads (test_gpu_fullsize.py runs them at the default 128)."""
import json
import random
from pathlib import Path

import numpy as np
import pytest

import fixtures as fx
import run_problems as rp
from oracle_compare import compare, set_modes
from run_problems import SMALL, Runs, unlimited, zonal_types, zone_names, zone_spread

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden" / "fullsize"
BLOCK_SIZES = (32, 128, 256, 512)


def closing_runs(seed):
    """Node types of 3 to 7 pods and runs of every size in rp.RUN_SIZES, alternating classes: a run first fills the open
    nodes with the fewest pods, wherever they sit in the active list, and closes the ones it brings to capacity."""
    rng = random.Random(seed)
    zs = zone_names(3, "sa-east")
    its = [t for cap in rng.sample((3, 4, 5, 7), 2) for t in zonal_types(zs, [(2, 4), (8, 32)], pods_cap=cap, prefix=f"c{cap}-")]
    r = Runs(f"close{seed}")
    reqs = ({"cpu": "100m", "memory": "64Mi"}, SMALL, {"cpu": "300m", "memory": "256Mi"})
    for i in range(14):
        k = rng.choice(rp.RUN_SIZES[:-1])
        if rng.random() < 0.4:
            r.run(f"spread-{i}", k, rng.choice(reqs), **zone_spread(f"spread-{i}", skew=rng.choice([1, 2])))
        else:
            r.run(f"plain-{i}", k, rng.choice(reqs), labels={"app": f"plain-{i}"})
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()])


@pytest.mark.parametrize("threads", BLOCK_SIZES)
@pytest.mark.parametrize("seed", (0, 1, 2))
def test_closing_runs_match_oracle(pkg, oracle, monkeypatch, seed, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    compare(pkg, oracle, pkg.Problem.from_dict(closing_runs(seed)))
    set_modes(monkeypatch)


def _full_size(pkg, cfg, pods, types, monkeypatch, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    problem = pkg.Problem.synth(cfg, pods, types, 42, 0)
    got = pkg.Scheduler(problem).solve(count_visited=False)
    set_modes(monkeypatch)
    return problem, got


def test_c2_full_size_at_512_threads(pkg, oracle, monkeypatch):
    problem, got = _full_size(pkg, 2, 10000, 500, monkeypatch, 512)
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    assert np.array_equal(got.assign, want.assign)
    assert got.digest() == want.digest()


@pytest.mark.parametrize("cfg,pods", [(3, 50000), (4, 100000)])
def test_c3_c4_full_size_at_512_threads(pkg, monkeypatch, cfg, pods):
    _, got = _full_size(pkg, cfg, pods, 1000, monkeypatch, 512)
    want = json.loads((GOLD / f"c{cfg}.json").read_text())
    assert np.array_equal(np.asarray(got.assign, dtype=np.int32), np.load(GOLD / f"c{cfg}_assign.npz")["assign"])
    assert got.num_new_nodes == want["new_nodes"]
    assert got.digest() == want["digest"]
