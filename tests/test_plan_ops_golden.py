"""CPU test: every DRY_RUN plan of tests/golden/make_plan_ops.py (C2C, R2C and both convolve plans; 1, 2, 3 and 8 devices;
P2P and NCCL; default, NO_FUSE and FORCE_FUSE; both directions and precisions; scaled, natural-spectrum, in-place, pipelined
and overlapped cases) records exactly the passes pinned by their SHA-256 in tests/golden/plan_ops.json.

On a mismatch, `python tests/golden/make_plan_ops.py KEY` prints the full records to diff against the parent's."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_plan_ops as mk  # noqa: E402


def test_plan_ops_match_the_golden(monkeypatch):
    for v in mk.SCHEDULE_ENV:
        monkeypatch.delenv(v, raising=False)
    with open(mk.OUT) as f:
        want = json.load(f)
    got = {mk.key(c): mk.digest(mk.record(c)) for c in mk.cases()}
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, "recorded schedules changed: %s" % bad[:20]
