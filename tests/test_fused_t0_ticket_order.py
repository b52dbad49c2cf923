"""Ticket order of the two-role t0 kernels (fft_fused2_kernel and fft_tma_fused_zy_kernel decode tickets through the same
fused2_decode).  Both kernels are deadlock free only if the order is a bijection onto the (role, plane, tile) triples and
every second-role (Y) tile of a plane is handed out after all first-role (Z) tiles of that plane: a Y tile waits for
exactly those, and a lower ticket is always held by a running CTA.  Checked on the host through the exported decode."""
import ctypes

import pytest

import distributedfft_b200 as dfft


@pytest.mark.parametrize("planes", [1, 2, 5, 24, 512])
@pytest.mark.parametrize("lag", range(9))
def test_ticket_order_is_a_bijection_and_respects_plane_dependencies(planes, lag):
    L = dfft.lib()
    out = (ctypes.c_longlong * 3)()
    GA, GB = 64, 64                      # 512-point fp64 planes, 8 lines / columns per tile
    if planes == 512 and lag not in (0, 3, 5, 8):
        GA, GB = 4, 3                    # keep the large case quick; unequal role sizes exercise the decode's strides
    total = L.dfft_debug_fused2_order(planes, GA, GB, lag, -1, out)
    assert total == planes * (GA + GB)
    seen = set()
    last_z = {}
    first_y = {}
    for t in range(total):
        assert L.dfft_debug_fused2_order(planes, GA, GB, lag, t, out) == total
        role, plane, idx = (int(x) for x in out)
        key = (role, plane, idx)
        assert key not in seen, key
        seen.add(key)
        assert role in (0, 1) and 0 <= plane < planes and 0 <= idx < (GA if role == 0 else GB), key
        if role == 0:
            last_z[plane] = t
        else:
            first_y.setdefault(plane, t)
    assert len(seen) == total
    for p in range(planes):
        assert last_z[p] < first_y[p], (p, last_z[p], first_y[p])


def test_ticket_order_runs_the_first_role_lag_planes_ahead():
    L = dfft.lib()
    out = (ctypes.c_longlong * 3)()
    planes, GA, GB, lag = 10, 4, 4, 3
    roles = []
    for t in range(L.dfft_debug_fused2_order(planes, GA, GB, lag, -1, out)):
        L.dfft_debug_fused2_order(planes, GA, GB, lag, t, out)
        roles.append((int(out[0]), int(out[1])))
    assert roles[: lag * GA] == [(0, p) for p in range(lag) for _ in range(GA)]
    assert roles[lag * GA: lag * GA + GA + GB] == [(0, lag)] * GA + [(1, 0)] * GB
    assert roles[-lag * GB:] == [(1, p) for p in range(planes - lag, planes) for _ in range(GB)]
