"""The training CorrBlock on the device (csrc/corr_train.cu through droid_slam_b200.modules.CorrBlock): every pyramid level, every call's
output and both feature-map gradients against the reference's formulation in fp64 on the same card (tests/corr_training_cases.py, held
to the unmodified reference's fixture here), within twice the error of that formulation's own fp32 execution (floor 2e-5 relative);
fnet's parameter gradients through install_corr_training_hook as DroidNet.forward calls it; fp32 lookups bit-identical to corr_index_forward; bit-reproducible backward;
no host synchronisation; the backward's peak memory; the forward-only checks on f16 maps that require grad."""
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from droid_slam_b200 import install, modules  # noqa: E402
from corr_training_cases import FIXTURE, RefCorrBlock, fixture_record, run  # noqa: E402
from corr_training_cases import make_inputs as _make_inputs  # noqa: E402
from util import host_syncs  # noqa: E402

pytestmark = pytest.mark.gpu

FLOOR = 2e-5          # relative to the largest magnitude of each compared tensor

# name: (B, N, ht, wd, calls, calls that feed the loss)
CASES = {
    "three_edges": (1, 3, 12, 16, 3, None),
    "odd_17x23": (1, 2, 17, 23, 3, None),
    "batch2": (2, 2, 9, 13, 2, None),
    "partial_loss": (1, 2, 16, 24, 4, (0, 2)),
    "wd_43x70": (1, 2, 43, 70, 2, None),
    "tiny_8x8": (1, 2, 8, 8, 2, None),
    "portrait_70x43": (1, 2, 70, 43, 2, None),
    "rows8_8x136": (1, 2, 8, 136, 2, None),
    "train_24x48x64": (1, 24, 48, 64, 15, None),
}


def reference_block(a, b):
    return RefCorrBlock(a, b)


def native_block(a, b):
    return modules.CorrBlock(a, b)


def make_inputs(*args, **kwargs):
    return _make_inputs(*args, dev="cuda", **kwargs)


def _err(x, t):
    return float((x.double() - t).abs().max()), float(t.abs().max())


@pytest.mark.parametrize("name", list(CASES))
def test_against_fp64_within_twice_the_reference_fp32_error(name):
    B, N, ht, wd, calls, used = CASES[name]
    f1, f2, coords, weights = make_inputs(B, N, ht, wd, calls)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        truth = run(reference_block, f1, f2, coords, weights, used, torch.float64)
        ref32 = run(reference_block, f1, f2, coords, weights, used, torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    nat = run(native_block, f1, f2, coords, weights, used, torch.float32)
    pairs = [("level %d" % l, nat[0][l], ref32[0][l], truth[0][l]) for l in range(4)]
    pairs += [("call %d" % k, nat[1][k], ref32[1][k], truth[1][k]) for k in range(calls)]
    pairs += [("grad fmap1", nat[2], ref32[2], truth[2]), ("grad fmap2", nat[3], ref32[3], truth[3])]
    for what, x, r, t in pairs:
        assert x.shape == t.shape and x.dtype == torch.float32, what
        e_nat, scale = _err(x, t)
        e_ref, _ = _err(r, t)
        assert e_nat <= max(2 * e_ref, FLOOR * scale), (name, what, e_nat, e_ref, scale)
    if used is not None:                       # calls outside the loss contribute nothing: same as a block that made only the used calls
        only = run(native_block, f1, f2, [coords[k] for k in used], [weights[k] for k in used], None, torch.float32)
        assert torch.equal(only[2], nat[2]) and torch.equal(only[3], nat[3])


@pytest.mark.parametrize("name", ["odd_17x23", "batch2", "wd_43x70", "tiny_8x8", "three_edges", "portrait_70x43", "rows8_8x136"])
def test_lookup_is_corr_index_forward_on_the_native_volume(name):
    B, N, ht, wd, calls, _ = CASES[name]
    be = install()
    f1, f2, coords, _ = make_inputs(B, N, ht, wd, calls, seed=1)
    with torch.no_grad():
        blk = modules.CorrBlock(f1, f2)
        for c in coords:
            got = blk(c)
            cc = c.permute(0, 1, 4, 2, 3).contiguous().view(B * N, 2, ht, wd)
            want = torch.cat([be.corr_index_forward(v, cc / 2 ** i, 3)[0].view(B, N, -1, ht, wd) for i, v in enumerate(blk.corr_pyramid)], 2)
            assert torch.equal(got, want)


def test_one_or_fifteen_calls_and_retained_graph_give_the_same_gradients():
    B, N, ht, wd, calls, _ = CASES["three_edges"]
    f1, f2, coords, weights = make_inputs(B, N, ht, wd, 15, seed=2)
    a, b = f1.clone().requires_grad_(True), f2.clone().requires_grad_(True)
    blk = modules.CorrBlock(a, b)
    outs = [blk(c) for c in coords]
    loss = sum((w * o).sum() for w, o in zip(weights, outs))
    first = torch.autograd.grad(loss, [a, b], retain_graph=True)
    second = torch.autograd.grad(loss, [a, b])
    assert torch.equal(first[0], second[0]) and torch.equal(first[1], second[1])
    again = run(native_block, f1, f2, coords, weights, None, torch.float32)     # a fresh block: bit-reproducible
    assert torch.equal(again[2], first[0]) and torch.equal(again[3], first[1])
    one = run(native_block, f1, f2, coords[:1], weights[:1], None, torch.float32)
    blk = modules.CorrBlock(a, b)
    outs = [blk(c) for c in coords]
    g = torch.autograd.grad((weights[0] * outs[0]).sum(), [a, b])
    assert torch.equal(g[0], one[2]) and torch.equal(g[1], one[3])


def test_no_host_sync_and_backward_memory_at_the_training_shape():
    B, N, ht, wd, calls, _ = CASES["train_24x48x64"]
    f1, f2, coords, weights = make_inputs(B, N, ht, wd, calls, seed=3)
    a, b = f1.clone().requires_grad_(True), f2.clone().requires_grad_(True)

    def step():
        blk = modules.CorrBlock(a, b)
        loss = sum((w * blk(c)).sum() for w, c in zip(weights, coords))
        loss.backward()
        return a.grad

    n, _ = host_syncs(step)
    assert n == 0
    a.grad = b.grad = None
    blk = modules.CorrBlock(a, b)
    loss = sum((w * blk(c)).sum() for w, c in zip(weights, coords))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    loss.backward()
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    q = sum((ht >> l) * (wd >> l) for l in range(4))
    gpyr_bytes = B * N * ht * wd * q * 4
    assert rise <= gpyr_bytes + 10 * f1.numel() * 4, (rise, gpyr_bytes, f1.numel() * 4)
    # the reference keeps no such bound: one dense gradient pyramid per call and level
    assert gpyr_bytes < 2 * sum(v.numel() for v in blk.corr_pyramid) * 4


def test_no_grad_keeps_nothing_for_backward():
    f1, f2, coords, _ = make_inputs(1, 2, 16, 24, 1, seed=4)
    a = f1.clone().requires_grad_(True)
    with torch.no_grad():
        blk = modules.CorrBlock(a, f2)
        out = blk(coords[0])
    assert blk._token is None and not out.requires_grad
    blk = modules.CorrBlock(f1, f2)
    assert blk._token is None and not blk(coords[0]).requires_grad


def test_f16_maps_that_require_grad_raise_in_both_hooks():
    f = torch.randn(1, 2, 128, 16, 24, device="cuda").half().requires_grad_(True)
    net = modules.install_corr_training_hook(types.SimpleNamespace(CorrBlock=lambda *a, **k: "reference"))
    with pytest.raises(RuntimeError, match="float16"):
        net.CorrBlock(f, f)
    assert modules.install_corr_training_hook(types.SimpleNamespace(CorrBlock=lambda *a, **k: "reference"), strict=False).CorrBlock(f, f) == "reference"

    class Ref:
        def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
            pass

    cls = modules.install_corr_volume_hook(types.SimpleNamespace(CorrBlock=type("CorrBlock", (Ref,), {}))).CorrBlock
    with pytest.raises(RuntimeError, match="forward only"):
        cls(f, f)
    with torch.no_grad():
        cls(f, f)                              # forward only under no_grad: builds natively


def test_fp64_truth_is_the_unmodified_reference():
    """the fp64 formulation the tests above take as truth, run on this card, against the reference's own fp64 run (the fixture)"""
    G = torch.load(os.path.join(ROOT, "tests", "golden", "corr_training.pt"))
    for name, (B, N, C, ht, wd, calls, used) in FIXTURE.items():
        f1, f2, coords, weights = make_inputs(B, N, ht, wd, calls, seed=11, C=C)
        rec = fixture_record(*run(RefCorrBlock, f1, f2, coords, weights, used, torch.float64))
        for k, want in G[name].items():
            assert float((rec[k].cpu() - want).abs().max()) <= 1e-12 * max(1.0, float(want.abs().max())), (name, k)


def test_fnet_gradients_through_the_hook_as_droidnet_calls_it():
    """DroidNet.forward's correlation path (droid_net.py:178-199): fnet on the frames, CorrBlock(fmaps[:,ii], fmaps[:,jj]) built through
    droid_net.CorrBlock, one lookup per update iteration at that iteration's coords1, a loss on every lookup -> fnet's parameter
    gradients, native hook against the reference's block in fp32, both against fp64"""
    import oracle.encoder as oenc
    from droid_slam_b200 import synth
    dev = "cuda"
    sd = synth.make_encoder_weights(0, 128)
    g = torch.Generator().manual_seed(21)
    images = torch.randn(1, 4, 3, 128, 160, generator=g)
    ii = torch.tensor([0, 1, 1, 2, 2, 3, 0, 3], device=dev)
    jj = torch.tensor([1, 0, 2, 1, 3, 2, 2, 1], device=dev)
    ht, wd, steps = 16, 20, 6
    y, x = torch.meshgrid(torch.arange(ht, dtype=torch.float32), torch.arange(wd, dtype=torch.float32), indexing="ij")
    coords1 = torch.stack([x, y], -1).expand(1, 8, ht, wd, 2) + 3 * torch.randn(1, 8, ht, wd, 2, generator=g)
    coords = []
    for _ in range(steps):                     # the update loop moves coords1 between lookups (detached, as droid_net.py:192-195)
        coords.append(coords1.to(dev))
        coords1 = coords1 + torch.randn(1, 8, ht, wd, 2, generator=g)
    weights = [torch.randn(1, 8, 196, ht, wd, generator=g).to(dev) for _ in range(steps)]

    def flow(native, dtype):
        params = {k: v.to(dev, dtype).requires_grad_(True) for k, v in sd.items()}
        droid_net = types.SimpleNamespace(CorrBlock=RefCorrBlock)
        if native:
            modules.install_corr_training_hook(droid_net)
        fmaps = oenc.encoder_forward(params, images.to(dev, dtype), "instance")
        corr_fn = droid_net.CorrBlock(fmaps[:, ii], fmaps[:, jj], num_levels=4, radius=3)
        if native:
            assert isinstance(corr_fn, modules.CorrBlock)
        loss = sum((w.to(dtype) * corr_fn(c)).sum() for w, c in zip(weights, coords))
        return dict(zip(params, torch.autograd.grad(loss, list(params.values()))))

    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        truth, ref32, nat = flow(False, torch.float64), flow(False, torch.float32), flow(True, torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    for k, t in truth.items():
        e_nat, scale = _err(nat[k], t)
        e_ref, _ = _err(ref32[k], t)
        assert scale > 0 and e_nat <= max(2 * e_ref, FLOOR * scale), (k, e_nat, e_ref, scale)
