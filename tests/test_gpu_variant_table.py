"""GPU: the pack kernel's variant table (csrc/pack_kernel.cuh, vt_build_entry), every fresh-node variant a class run can
replay, built in the row gather's launch before the pack kernel. The run, shape, run-variant, round-stretch and
fill-stretch corpora are compared with the oracle on the whole result with the table on and off (KSCHED_NO_VARSTORE) at
32 / 128 / 512 threads, and with the table on under each mode switch; so are the table's own near misses
(tests/variant_table_problems.py), each of which must take its variants from the table or not at all, as it was built
to. Every corpus must reach the table; C4 must take every variant from it, with no derivation left."""
import json
from pathlib import Path

import numpy as np
import pytest

import fill_stretch_problems as fsp
import round_stretch_problems as rsp
import run_problems as rp
import run_variant_problems as rvp
import shape_problems as sp
import variant_table_problems as vt
from oracle_compare import MODE_SWITCHES, set_modes

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / "golden" / "fullsize"
CORPORA = [("table", vt, c) for c in vt.CORPUS] + [("shape", sp, c) for c in sp.CORPUS] + [("runvar", rvp, c) for c in rvp.CORPUS] + \
          [("round", rsp, c) for c in rsp.CORPUS] + [("fill", fsp, c) for c in fsp.CORPUS] + [("run", rp, c) for c in rp.CORPUS]


def _resident(pkg, problem):
    rs = pkg.ResidentSolve(problem)
    rs.set_count_visited(False)
    rs.load()
    return rs


def _problem(pkg, mod, name, seed):
    built = mod.build(name, seed)
    return pkg.Problem.from_dict(built[0] if isinstance(built, tuple) else built)


@pytest.mark.parametrize("corpus,mod,case", CORPORA, ids=[f"{k}-{c[0]}-{c[1]}" for k, _, c in CORPORA])
def test_table_on_and_off_match_oracle(pkg, oracle, monkeypatch, corpus, mod, case):
    problem = _problem(pkg, mod, *case)
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    rs = _resident(pkg, problem)
    for table in ("on", "off"):
        for threads in (32, 128, 512):
            monkeypatch.setenv("KSCHED_PACK_THREADS", str(threads))
            if table == "off":
                monkeypatch.setenv("KSCHED_NO_VARSTORE", "1")
            else:
                monkeypatch.delenv("KSCHED_NO_VARSTORE", raising=False)
            rs.run()
            res = rs.download()
            assert (res.assign == want.assign).all(), (table, threads)
            assert res.digest() == want.digest(), (table, threads)
            t = rs.timings()
            if table == "off":
                assert t["vt_fetches"] == 0


SWITCHES = tuple(m for m in MODE_SWITCHES if m != "KSCHED_NO_VARSTORE") + ("KSCHED_NO_RUNDERIVE",)


@pytest.mark.parametrize("corpus,mod,case", CORPORA, ids=[f"{k}-{c[0]}-{c[1]}" for k, _, c in CORPORA])
def test_table_under_each_switch_matches_oracle(pkg, oracle, monkeypatch, corpus, mod, case):
    problem = _problem(pkg, mod, *case)
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    rs = _resident(pkg, problem)
    for switch in SWITCHES:
        set_modes(monkeypatch, switch)
        monkeypatch.delenv("KSCHED_NO_RUNDERIVE", raising=False)
        if switch == "KSCHED_NO_RUNDERIVE":
            monkeypatch.setenv(switch, "1")
        rs.run()
        res = rs.download()
        assert (res.assign == want.assign).all(), switch
        assert res.digest() == want.digest(), switch
    set_modes(monkeypatch)
    monkeypatch.delenv("KSCHED_NO_RUNDERIVE", raising=False)


def _counts(pkg, mod, case):
    rs = _resident(pkg, _problem(pkg, mod, *case))
    rs.run()
    rs.download()
    t = rs.timings()
    return t["vt_fetches"], t["run_derives"]


@pytest.mark.parametrize("mod", [sp, rvp, rsp, fsp, rp], ids=lambda m: m.__name__)
def test_each_corpus_reaches_the_table(pkg, monkeypatch, mod):
    set_modes(monkeypatch)
    assert sum(_counts(pkg, mod, case)[0] for case in mod.CORPUS) > 0


@pytest.mark.parametrize("name,seed", vt.CORPUS, ids=[f"{n}-{s}" for n, s in vt.CORPUS])
def test_near_miss_reach(pkg, monkeypatch, name, seed):
    """"table": the runs fetch entries and derive nothing; "none": no entry is fetched and the runs derive their variants;
    "both": the covered classes fetch, the others derive"""
    set_modes(monkeypatch)
    monkeypatch.delenv("KSCHED_NO_RUNDERIVE", raising=False)
    fetches, derives = _counts(pkg, vt, (name, seed))
    reach = vt.build(name, seed)[1]["reach"]
    if reach == "table":
        assert fetches > 0 and derives == 0, (fetches, derives)
    elif reach == "none":
        assert fetches == 0 and derives > 0, (fetches, derives)
    else:
        assert fetches > 0 and derives > 0, (fetches, derives)


def test_c4_takes_every_variant_from_the_table(pkg, monkeypatch):
    monkeypatch.delenv("KSCHED_NO_VARSTORE", raising=False)
    rs = _resident(pkg, pkg.Problem.synth(4, 100000, 1000, 42, 0))
    rs.run()
    res = rs.download()
    t = rs.timings()
    want = json.loads((GOLD / "c4.json").read_text())
    assert np.array_equal(np.asarray(res.assign, dtype=np.int32), np.load(GOLD / "c4_assign.npz")["assign"])
    assert res.digest() == want["digest"]
    assert t["vt_fetches"] > 0 and t["run_derives"] == 0, t
    assert t["vt_build_us"] > 0, t


def test_shape_corpus_reaches_the_table(pkg, monkeypatch):
    """Deployments of one shape take their fresh nodes from the table; the near misses the table does not cover
    (volumes, instance-type or hostname requirements) still derive theirs, as they did without it."""
    counts = {}
    for table in ("on", "off"):
        if table == "off":
            monkeypatch.setenv("KSCHED_NO_VARSTORE", "1")
        else:
            monkeypatch.delenv("KSCHED_NO_VARSTORE", raising=False)
        fetches = derives = 0
        for case in sp.CORPUS:
            rs = _resident(pkg, _problem(pkg, sp, *case))
            rs.run()
            rs.download()
            t = rs.timings()
            fetches += t["vt_fetches"]
            derives += t["run_derives"]
        counts[table] = (fetches, derives)
    assert counts["on"][0] > 0 and counts["off"][0] == 0, counts
    assert counts["on"][1] < counts["off"][1], counts
