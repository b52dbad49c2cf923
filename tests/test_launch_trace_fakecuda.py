"""CPU test: non-dry C2C, R2C and convolve plans issue exactly the launch traces pinned in tests/golden/launch_traces.json.

The library's objects run against tests/fakecuda/fake_cudart.cpp, which logs per host thread, in issue order, every kernel
launch (device name, grid, block, dynamic shared memory, stream, and the start gate / completion signal a pass kernel carries),
every flag kernel's word and epoch, every event record and stream wait, and every async copy and set.  Plans of 1, 2 and 4
device-threads (P2P) run two executes each, without TMA, with the TMA stand-in (FAKECUDA_TMA=1) and with every TMA pass mode on
(DFFT_TMA=2).  This pins what DRY_RUN records cannot see: the order of the gate and signal kernels relative to the passes, which
pass carries a folded signal, and the timing event brackets.  The NCCL schedules need a real NCCL and are pinned by the DRY_RUN
digests (tests/golden/plan_ops.json) only.

On a mismatch, `python tests/golden/make_launch_traces.py --show KEY` prints the full traces to diff against the parent's."""
import json
import os
import sys

import pytest

from test_control_flow_fakecuda import ROOT, fake_lib  # noqa: F401  (fixture)

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_launch_traces as mk  # noqa: E402


@pytest.mark.parametrize("flavour", list(mk.FLAVOURS))
def test_launch_traces_match_the_golden(fake_lib, flavour):  # noqa: F811
    with open(mk.OUT) as f:
        want = {k: v for k, v in json.load(f).items() if k.startswith(flavour + ":")}
    got = {k: [mk.digest(lines) for lines in per_thread] for k, per_thread in mk.traces(fake_lib, flavour).items()}
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, "launch traces changed: %s" % bad[:20]
