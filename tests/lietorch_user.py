"""A module that imports `lietorch` at import time, as the reference's depth_video does, with a backend_process global: the spawned-child
test of tests/test_lietorch_cpu.py starts a DroidAsync-style Process on it whose argument is a Holder of this module."""
import sys

import lietorch

LIETORCH = lietorch.__name__


class Holder:
    """an argument whose unpickling imports this module, and so `lietorch`"""


def backend_process(holder, queue, unused=None, device="cuda"):
    """the module's own backend_process (what install_async_hook(strict=False) runs in a child without the native backend's hooks)"""
    queue.put((LIETORCH, sys.modules["lietorch"].__name__, sys.modules["torch_scatter"].__name__))
