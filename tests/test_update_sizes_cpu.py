"""dba_update_workspace_bytes (host only): unchanged where wd % 8 == 0, where the convolutions keep their rectangular tiles, and large
enough for the row-flattened tiles' partial-sum slots elsewhere.  The expected values are those of the build before row-flattened
tiles existed."""
import pytest

from droid_slam_b200 import c_api


@pytest.fixture(scope="module")
def ws_bytes():
    return c_api.load().dba_update_workspace_bytes


@pytest.mark.parametrize("shape,expected", [
    ((512, 72, 48, 64), 5700848384), ((6, 3, 16, 64), 23406080), ((5, 4, 24, 32), 15220736), ((3, 2, 10, 40), 4747776),
    ((1, 0, 30, 40), 4933120), ((100, 10, 72, 96), 2490686208), ((4, 2, 8, 8), 1030656), ((512, 72, 30, 40), 2255162112),
    ((64, 8, 44, 72), 737575680),
])
def test_workspace_unchanged_at_widths_that_are_multiples_of_8(ws_bytes, shape, expected):
    assert ws_bytes(*shape) == expected


@pytest.mark.parametrize("E,n_src,ht,wd", [(512, 72, 43, 70), (512, 72, 44, 69), (512, 72, 41, 73), (6, 3, 9, 13), (1, 1, 1, 1), (2, 1, 12, 157)])
def test_workspace_holds_row_flattened_gate_slots(ws_bytes, E, n_src, ht, wd):
    """the EPI_GATE partial sums: E x slots x 128 floats, slots = 8 per linear M tile, at most ceil(ht * pitch / 128) + 3 M tiles"""
    pitch = (wd + 7) // 8 * 8
    slots = ((ht * pitch + 127) // 128 + 3) * 8
    px = E * ht * wd
    activations = px * 2 * (128 + 320 + 200 + 200 + 128 * 4 + 384)          # the channels-last buffers before the partial sums
    assert ws_bytes(E, n_src, ht, wd) >= activations + E * slots * 128 * 4
