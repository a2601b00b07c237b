"""The reference's own Python, imported unmodified by the golden generators and the live CPU checks.

`REF` is the reference checkout (DROID_REFERENCE_ROOT, default /root/reference); this module imports without it, and no GPU test reads
it.  `reference_modules` imports the reference's droid_slam modules on the pure-PyTorch stand-ins of oracle/shims and leaves sys.path
and sys.modules as it found them; `cuda_on_cpu` serves the reference's hard-coded "cuda" on the CPU."""
import contextlib
import importlib
import os
import sys

import torch

from oracle.shims import lietorch as _lietorch, torch_scatter as _torch_scatter

REF = os.path.abspath(os.environ.get("DROID_REFERENCE_ROOT", "/root/reference"))


def present(*parts):
    """whether REF/<parts> exists"""
    return os.path.exists(os.path.join(REF, *parts))


@contextlib.contextmanager
def reference_modules(*names, stubs=None):
    """yields the modules `names` (dotted, under droid_slam/) imported unmodified, with `lietorch` / `torch_scatter` the stand-ins and
    `stubs` ({name: module}) in sys.modules.  On exit sys.path is restored, every stubbed name is restored or removed, and every module
    imported from REF is removed, so that no later import finds them; the modules taken out of the block keep working through the names
    they bound at import."""
    stubs = {"lietorch": _lietorch, "torch_scatter": _torch_scatter, **(stubs or {})}
    path, before = list(sys.path), dict(sys.modules)
    sys.modules.update(stubs)
    sys.path.insert(0, os.path.join(REF, "droid_slam"))
    try:
        yield tuple(importlib.import_module(name) for name in names)
    finally:
        sys.path[:] = path
        for name in stubs:
            if name in before:
                sys.modules[name] = before[name]
            else:
                sys.modules.pop(name, None)
        under = os.path.join(REF, "")
        for name, m in list(sys.modules.items()):
            if name not in before and (getattr(m, "__file__", None) or "").startswith(under):
                del sys.modules[name]


@contextlib.contextmanager
def cuda_on_cpu():
    """inside the block Tensor.cuda() is the identity and torch.as_tensor(..., device="cuda...") lands on the CPU"""
    cuda, as_tensor = torch.Tensor.cuda, torch.as_tensor

    def on_cpu(data, dtype=None, device=None):
        return as_tensor(data, dtype=dtype, device="cpu" if str(device).startswith("cuda") else device)

    torch.Tensor.cuda, torch.as_tensor = (lambda self, *a, **k: self), on_cpu
    try:
        yield
    finally:
        torch.Tensor.cuda, torch.as_tensor = cuda, as_tensor
