"""The host encoder's output (every byte handed to the C-ABI) for a fixed corpus must match the committed digests:
encoder refactors are proven result-neutral here, on the CPU. Regenerate with tests/golden/make_encoding_digests.py after an
intended change of the encoding."""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests" / "golden"))


def test_encoder_output_matches_committed_digests(pkg):
    import make_encoding_digests as m
    want = json.loads((ROOT / "tests" / "golden" / "encoding_digests.json").read_text())
    got = {name: m.digest(pkg, problem, cands, superset) for name, problem, cands, superset in m.corpus(pkg)}
    assert set(got) == set(want)
    wrong = [n for n in got if got[n] != want[n]]
    assert not wrong, wrong[:10]
