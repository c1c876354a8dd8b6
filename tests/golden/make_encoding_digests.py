"""Regenerates tests/golden/encoding_digests.json: a digest (kh_encoded_digest) of everything the host encoder hands to the
C-ABI, for a corpus of problems. The encoder is the one piece of the product that is pure host code on the GPU path, so a
refactor / speed-up of it can be proven result-neutral on the CPU: same bytes in, same kernels, same results.
Run after any INTENDED change of the encoding (new catalog field, different dictionary order, ...):
    python tests/golden/make_encoding_digests.py
"""
import ctypes as C
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def corpus(pkg):
    """(name, problem, candidates, cluster_superset): cluster_superset digests the encoding ksched_load_cluster takes"""
    import consolidation_answers as ca
    import extended_resource_problems as xp
    import known_answers as ka
    import itertools
    import provisioner_problems as pp
    import round_stretch_problems as rsp
    import run_problems as rp
    import shape_problems as sp
    import taint_problems as tp
    import validation_problems as vp
    import wide_problems as wp

    import fixtures as fx
    from fuzz_problems import random_problem, random_problem_with_bounds

    def fresh():  # pod names / uids come from a process-wide counter in the fixtures: restart it so the corpus does not depend on test order
        fx._uid = itertools.count()

    def cluster(name, problem, pd):  # the candidates marked in the problem, in list order and reversed
        cands = tuple(j for j, n in enumerate(pd.get("nodes", [])) if n.get("candidate"))
        yield f"cluster-{name}", problem, cands, True
        if len(cands) > 1:
            yield f"cluster-{name}-rev", problem, cands[::-1], True

    def both(name, pd):  # a feature test's problem: its plain and its superset encodings
        name = f"feature-{name}"
        problem = pkg.Problem.from_dict(pd)
        yield name, problem, (), False
        yield from cluster(name, problem, pd)

    for seed in range(300):
        fresh()
        yield f"fuzz-{seed}", pkg.Problem.from_dict(random_problem(seed)), (), False
    for name, _, build in ka.CASES + ka.CPU_ONLY_CASES + ca.CASES + ca.CPU_ONLY_CASES:
        fresh()
        prob, _ = build()
        for i, pd in enumerate(prob["multi"] if "multi" in prob else [prob]):
            problem = pkg.Problem.from_dict(pd)
            yield f"ka-{name}-{i}", problem, (), False
            n_cand = sum(1 for n in pd.get("nodes", []) if n.get("candidate"))
            for c in range(1, n_cand + 1):
                yield f"ka-{name}-{i}-cand{c}", problem, tuple(j for j, n in enumerate(pd["nodes"]) if n.get("candidate"))[:c], False
            if pd.get("nodes"):
                yield from cluster(f"ka-{name}-{i}", problem, pd)
    for cfg, pods, types, nodes in ((1, 100, 10, 0), (2, 3000, 500, 0), (3, 3000, 1000, 0), (4, 3000, 1000, 0), (5, 2000, 1000, 200)):
        problem = pkg.Problem.synth(cfg, pods, types, 42, nodes)
        yield f"synth-{cfg}", problem, (), False
        if cfg == 5:
            for c in (1, 2, 17, 100, 199):
                yield f"synth-5-cand{c}", problem, tuple(range(c)), False
                yield f"cluster-synth-5-cand{c}", problem, tuple(range(c)), True

    # the feature corpora: wide label keys, many provisioners, many taint sets, ext resources, the pack kernel's run shapes
    for prefix, make in (("wide", wp.corpus), ("prov", pp.corpus), ("taint", tp.corpus), ("ext", xp.corpus), ("ext", xp.fresh_corpus)):
        fresh()
        for name, pd, *_ in make():
            yield from both(f"{prefix}-{name}", pd)
    for name, make in (("ext-too-many-resources", xp.too_many_resources), ("ext-too-many-slot-resources", xp.too_many_slot_resources)):
        fresh()
        yield from both(name, make())
    for prefix, mod in (("run", rp), ("shape", sp), ("stretch", rsp)):
        for name, seed in mod.CORPUS:
            fresh()
            yield from both(f"{prefix}-{name}-{seed}", mod.build(name, seed)[0])
    fresh()
    for name, before, after in vp.pairs():
        yield from both(f"validation-{name}-before", before)
        yield from both(f"validation-{name}-after", after)
    for seed in range(70):
        fresh()
        yield from both(f"bounds-{seed}", random_problem_with_bounds(seed))
    # consolidation clusters of the feature modules, and the same clusters after the TTL
    for name, make in (("prov-cluster", pp.cluster), ("prov-after", pp.after), ("taint-cluster", tp.cluster), ("taint-after", tp.after),
                       ("ext-cluster", xp.cluster), ("ext-after", xp.after), ("wide-cluster", wp.cluster)):
        fresh()
        yield from both(f"{name}-0", make(0))
    for seed, zones, ct_spread in ((1, 9, False), (2, 16, False), (3, 9, True)):
        fresh()
        yield from both(f"run-cluster-{seed}-{zones}-{int(ct_spread)}", rp.cluster(seed, zones, ct_spread))


def digest(pkg, problem, candidates, cluster_superset=False):
    arr = (C.c_int * max(1, len(candidates)))(*candidates)
    encode = pkg.lib().kh_encode_cluster if cluster_superset else pkg.lib().kh_encode
    enc = encode(problem.ptr, arr, len(candidates))
    if not enc:
        return "refused: " + pkg.lib().kh_scheduler_error().decode()[:80]
    d = pkg.lib().kh_encoded_digest(enc)
    pkg.lib().kh_encoded_free(enc)
    return f"{d:016x}"


def main():
    import __graft_entry__ as g
    pkg = g.load_pkg()
    out = {}
    for name, problem, cands, superset in corpus(pkg):
        assert name not in out, name
        out[name] = digest(pkg, problem, cands, superset)
    (ROOT / "tests" / "golden" / "encoding_digests.json").write_text(json.dumps(out, indent=0, sort_keys=True) + "\n")
    print(len(out), "digests written")


if __name__ == "__main__":
    main()
