"""Records the executed reference's answers for the tests that compare against it (tests/ref_replay.py) into
tests/golden/live_ref_vectors.npz.  Needs the reference binaries under oracle/_ref, which build() compiles from the
reference tree when that tree is present:

    python tests/golden/make_live_ref_vectors.py
"""
import os
import sys

import pytest

TESTS = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, TESTS)
sys.path.insert(0, os.path.dirname(TESTS))

import ref_replay  # noqa: E402
from oracle import build_ref, build_ref3d  # noqa: E402

if __name__ == "__main__":
    assert build_ref() is not None and build_ref3d() is not None, "the reference binaries under oracle/_ref are missing"
    store = {}
    ref_replay.RECORDING["store"] = store
    rc = pytest.main(["-q", "-p", "no:cacheprovider", os.path.join(TESTS, "test_oracle_ref.py"), os.path.join(TESTS, "test_oracle_ref3d.py"),
                      os.path.join(TESTS, "test_control_flow_fakecuda.py") + "::test_driver_stdout_surface_is_the_reference_drivers"])
    assert rc == 0, rc
    ref_replay.save(store)
    print("wrote", ref_replay.PATH, os.path.getsize(ref_replay.PATH), "bytes")
