"""CPU test: the lines engine (dfft_lines_* plans) still describes and launches exactly what tests/golden/make_lines_goldens.py
pinned: the records of the five dfft_debug_lines*_ops hooks, or their return codes for rejected specs
(tests/golden/lines_plan_ops.json), and the fake-runtime launch trace of every lines create entry point
(tests/golden/lines_launch_traces.json; its worker also checks that no plan leaves an allocation behind).

On a mismatch, `python tests/golden/make_lines_goldens.py --show KEY` prints the records and traces to diff against the parent's."""
import json
import os
import sys

from test_control_flow_fakecuda import ROOT, fake_lib  # noqa: F401  (fixture)

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_lines_goldens as mk  # noqa: E402


def test_lines_plan_ops_match_the_golden(monkeypatch):
    for v in mk.LINES_ENV:
        monkeypatch.delenv(v, raising=False)
    with open(mk.OPS_OUT) as f:
        want = json.load(f)
    got = mk.plan_ops()
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, "lines records changed: %s" % bad[:20]


def test_lines_launch_traces_match_the_golden(fake_lib):  # noqa: F811
    with open(mk.TRACES_OUT) as f:
        want = json.load(f)
    got = {k: mk.digest(lines) for k, lines in mk.launch_traces(fake_lib).items()}
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, "lines launch traces changed: %s" % bad[:20]
