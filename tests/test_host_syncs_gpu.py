"""The measuring helpers of tests/util.py that the GPU tests and the bench tools share: host_syncs counts exactly the synchronising
operations, also in a process's first counting window; syncs_not_counted hides a sync from it; both give back the debug mode they
found; card() reads the device torch is using."""
import json
import os
import subprocess
import sys

import pytest
import torch

from util import card, host_syncs, syncs_not_counted

pytestmark = pytest.mark.gpu
TESTS = os.path.dirname(os.path.abspath(__file__))

# the process's first two counting windows: device work with no sync, then one .item()
FIRST_WINDOWS = """
import json, sys
sys.path.insert(0, %r)
import torch
from util import host_syncs
x = torch.arange(1000, device="cuda", dtype=torch.float32)
none, _ = host_syncs(lambda: (x * 2).sum())
one, v = host_syncs(lambda: x.sum().item())
print(json.dumps([none, one, v]))
""" % TESTS


def test_first_windows_of_a_process():
    r = subprocess.run([sys.executable, "-c", FIRST_WINDOWS], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert json.loads(r.stdout.strip().splitlines()[-1]) == [0, 1, 499500.0]


@pytest.mark.parametrize("before", [0, 1])
def test_syncs_not_counted_and_the_mode_restored(before):
    x = torch.ones(16, device="cuda")

    def hidden():
        with syncs_not_counted():
            x.sum().item()
        assert torch.cuda.get_sync_debug_mode() == 1

    def raises():
        with syncs_not_counted():
            raise ValueError("inside")

    torch.cuda.set_sync_debug_mode(before)
    try:
        assert host_syncs(hidden)[0] == 0
        assert torch.cuda.get_sync_debug_mode() == before
        with pytest.raises(ValueError, match="inside"):
            host_syncs(raises)
        assert torch.cuda.get_sync_debug_mode() == before
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_card_is_the_current_device():
    c = card()
    assert c["name"] == torch.cuda.get_device_name(), c
    assert not c["power_limit"].startswith("unknown"), c
