"""GPU differential fuzz: random problems mixing every feature; the CUDA path must equal the oracle bit-for-bit, or refuse
loudly with KSCHED_ERR_UNSUPPORTED (never a silently different answer)."""
import pytest

from fuzz_problems import random_problem, random_problem_with_bounds
from oracle_compare import compare

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", range(150))
def test_gpu_equals_oracle_with_gt_lt_and_complement_types(pkg, oracle, seed):
    """Gt / Lt requirements and complement instance-type requirements (region form on the device)"""
    _compare(pkg, oracle, random_problem_with_bounds(seed))


@pytest.mark.parametrize("seed", range(300))
def test_gpu_equals_oracle_on_random_problem(pkg, oracle, seed):
    _compare(pkg, oracle, random_problem(seed))


def _compare(pkg, oracle, prob):
    compare(pkg, oracle, pkg.Problem.from_dict(prob), add_calls=False, refusal_skips=True)
