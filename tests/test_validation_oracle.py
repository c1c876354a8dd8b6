"""CPU: consolidation validation on the oracle - the known answers, fast mode against the literal path on the corpus, and
the single-node sweep split into shares merging to the whole sweep."""
import pytest

import validation_answers as va
import validation_oracle as vo
import validation_problems as vp


def _pp(pkg, d):
    return d, pkg.Problem.from_dict(d)


@pytest.mark.parametrize("name,ref,build", va.CASES, ids=[c[0] for c in va.CASES])
def test_known_answer_on_the_oracle(pkg, oracle, name, ref, build):
    (b, a), check = build()
    before, after = _pp(pkg, b), _pp(pkg, a)
    check(vo.single_compute_command(before, after), vo.multi_compute_command(before, after))


def test_corpus_exercises_both_verdicts(pkg, oracle):
    seen = set()
    for name, b, a in vp.pairs()[::4]:
        r = vo.single_compute_command(_pp(pkg, b), _pp(pkg, a))
        seen.update(v for _, v in r["validations"])
        seen.add(r["action"])
    assert {True, False, 3} <= seen


def test_fast_mode_equals_the_literal_path(pkg, oracle):
    for name, b, a in vp.pairs()[::3]:
        before, after = _pp(pkg, b), _pp(pkg, a)
        try:
            oracle.lib.oracle_set_fast(0)
            lit = (vo.single_compute_command(before, after), vo.multi_compute_command(before, after))
            oracle.lib.oracle_set_fast(1)
            fast = (vo.single_compute_command(before, after), vo.multi_compute_command(before, after))
        finally:
            oracle.lib.oracle_set_fast(0)
        assert lit == fast, name


def test_single_node_shares_merge_to_the_whole_sweep(pkg, oracle):
    for name, b, a in vp.pairs()[::5]:
        before, after = _pp(pkg, b), _pp(pkg, a)
        whole = vo.single_compute_command(before, after)
        n = len(oracle.rank_candidates(before[1])[0])
        half = n // 2
        merged = pkg.merge_single_node_shares([vo.single_compute_command(before, after, 0, half),
                                               vo.single_compute_command(before, after, half, -1)])
        keys = ("action", "position", "node", "options", "validations", "failed_validation")
        assert {k: merged[k] for k in keys} == {k: whole[k] for k in keys}, name
