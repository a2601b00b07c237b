"""droid_slam_b200.lietorch / torch_scatter and install_dependencies() without a GPU: the gradient-convention oracle (oracle/lie_grad.py)
against the closed forms of lietorch's backward kernels, the package's construction / indexing / cat on CPU tensors and the wording of
its refusals, the registration of both modules (also in a spawned DroidAsync-style child), and torch_scatter's known answers."""
import contextlib
import multiprocessing
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import droid_slam_b200  # noqa: E402
from droid_slam_b200 import lietorch as lt, modules, torch_scatter as ts  # noqa: E402
from oracle import lie_grad as lg  # noqa: E402

F64 = torch.float64


def _case(group, op, seed):
    g = torch.Generator().manual_seed(seed)
    G = lg.cls(group)
    K, N = G.manifold_dim, G.embedded_dim
    a = 0.8 * torch.randn(6, K, generator=g, dtype=F64)
    X = G.exp(torch.randn(6, K, generator=g, dtype=F64)).data
    A = a if op == "exp" else X
    B = {"mul": G.exp(torch.randn(6, K, generator=g, dtype=F64)).data, "adj": a, "adjT": a, "act": torch.randn(6, 3, generator=g, dtype=F64),
         "act4": torch.randn(6, 4, generator=g, dtype=F64)}.get(op)
    n = {"exp": N, "inv": N, "mul": N, "fromvec": N, "vec": N, "log": K, "adj": K, "adjT": K, "act": 3, "act4": 4}[op]
    u = torch.randn(6, n, generator=g, dtype=F64)
    if op in lg.GROUP_OUT:
        u[:, K:] = 0
    return A, B, u


def _diff(r1, r2):
    return max(float((x - y).abs().max()) for x, y in zip(r1, r2) if x is not None)


@pytest.mark.parametrize("group", ["SO3", "SE3"])
@pytest.mark.parametrize("op", lg.OPS)
def test_oracle_agrees_with_the_closed_forms(group, op):
    A, B, u = _case(group, op, 1)
    assert _diff(lg.autograd_grad(group, op, A, B, u), lg.closed_grad(group, op, A, B, u)) < 1e-12


@pytest.mark.parametrize("group", ["SO3", "SE3"])
@pytest.mark.parametrize("op", [o for o in lg.OPS if o not in ("exp", "fromvec")])
def test_oracle_rejects_a_right_perturbation_and_a_transpose(group, op):
    A, B, u = _case(group, op, 2)
    closed = lg.closed_grad(group, op, A, B, u)
    assert _diff(lg.autograd_grad(group, op, A, B, u, perturb="right"), closed) > 1e-3
    assert _diff(lg.autograd_grad(group, op, A, B, u), lg.closed_grad(group, op, A, B, u, transposed=True)) > 1e-3


def test_first_order_exponential_matches_the_stand_ins_exp():
    for G in (lg.shim.SO3, lg.shim.SE3):
        e = torch.randn(5, G.manifold_dim, dtype=F64)
        for s in (1e-3, 1e-4):
            assert float((lg.exp1(G, s * e).data - G.exp(s * e).data).abs().max()) < 10 * s * s


def test_package_on_the_cpu():
    """construction, Identity, indexing, cat and stack give the stand-in's data; CPU and Sim3 / RxSO3 arithmetic raise"""
    assert set(lt.__all__) == {"LieGroupParameter", "SO3", "RxSO3", "SE3", "Sim3", "cat", "stack"}
    S = lg.shim
    data = S.SE3.exp(torch.randn(2, 5, 6, dtype=F64)).data
    X, Xs = lt.SE3(data), S.SE3(data)
    assert torch.equal(lt.SE3.Identity(2, 3).data, S.SE3.Identity(2, 3).data) and lt.SE3.Identity(1).data.dtype == torch.float32
    assert torch.equal(lt.SE3.Identity(1,).data.squeeze(), torch.tensor([0.0, 0, 0, 0, 0, 0, 1]))      # motion_filter.py:55
    assert torch.equal(lt.SO3.IdentityLike(lt.SO3(X)).data, S.SO3.Identity(2, 5, dtype=F64).data)
    assert torch.equal(X[:, torch.tensor([0, 2])].data, Xs[:, torch.tensor([0, 2])].data) and X[:, :, None, None].data.shape == (2, 5, 1, 1, 7)
    assert torch.equal(lt.cat([X, X], 1).data, S.cat([Xs, Xs], 1).data) and torch.equal(lt.stack([X, X], 0).data, S.stack([Xs, Xs], 0).data)
    assert X.shape == (2, 5) and X.tangent_shape == (2, 5, 6) and X.dtype == F64 and X.device.type == "cpu"
    assert torch.equal(lt.SO3(X).data, data[..., 3:]) and torch.equal(lt.SE3(lt.SO3(X)).data[..., :3], torch.zeros(2, 5, 3, dtype=F64))
    Y = X.view((10,))
    Y[3] = lt.SE3.Identity(1, dtype=F64)[0]
    assert torch.equal(data.view(10, 7)[3], lt.SE3.id_elem.double()) and len(X.unbind(1)) == 5
    assert torch.equal(X.vec(), data) and isinstance(lt.SE3.InitFromVec(data), lt.SE3)
    for f, name in ((lambda: X.inv(), "SE3.inv"), (lambda: X.log(), "SE3.log"), (lambda: lt.SE3.exp(torch.zeros(6)), "SE3.exp"),
                    (lambda: X * X, "SE3.mul"), (lambda: X.act(torch.zeros(2, 5, 3, dtype=F64)), "SE3.act"), (lambda: X.matrix(), "SE3.matrix")):
        with pytest.raises(RuntimeError, match="^%s has no kernel for this call: a cpu tensor" % name):
            f()
    Z = lt.Sim3(X)
    assert isinstance(Z, lt.Sim3) and Z.data.shape == (2, 5, 8) and torch.equal(lt.RxSO3(Z).data, torch.cat([data[..., 3:], torch.ones(2, 5, 1, dtype=F64)], -1))
    assert torch.equal(lt.cat([Z, Z], 0).data, torch.cat([Z.data, Z.data])) and isinstance(Z[0], lt.Sim3)
    for f, name in ((lambda: Z.inv(), "Sim3.inv"), (lambda: Z * Z, "Sim3.mul"), (lambda: lt.Sim3.exp(torch.zeros(7)), "Sim3.exp"),
                    (lambda: lt.RxSO3(Z).log(), "RxSO3.log"), (lambda: Z.act(torch.zeros(2, 5, 3)), "Sim3.act")):
        with pytest.raises(RuntimeError, match="^%s has no kernel for this call: .*arithmetic is not implemented" % name):
            f()


@contextlib.contextmanager
def registered_state():
    """sys.modules' lietorch / torch_scatter and the hook registry restored after the block (install_dependencies registers both)"""
    saved = {k: sys.modules.get(k) for k in ("lietorch", "torch_scatter")}
    hooks = list(modules._HOOKS)
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        modules._HOOKS[:] = hooks


def test_install_dependencies_registers_refuses_to_shadow_and_leaves_install_alone():
    with registered_state():
        be = droid_slam_b200.install()
        assert "lietorch" not in sys.modules and "torch_scatter" not in sys.modules          # install() does not register them
        assert droid_slam_b200.install_dependencies() is be
        import lietorch
        import torch_scatter
        from lietorch import SE3
        assert lietorch is lt and torch_scatter is ts and SE3 is lt.SE3
        assert [e["installer"] for e in modules.hook_registry()][-1] == "install_dependencies"
        assert modules.hook_registry()[-1]["transferable"] and modules.hook_registry()[-1]["module"] == "droid_slam_b200"
        droid_slam_b200.install_dependencies()                                               # again: the same modules, no error
        sys.modules["lietorch"] = types.ModuleType("lietorch")
        with pytest.raises(ImportError, match="a different `lietorch` module is already imported"):
            droid_slam_b200.install_dependencies()
        sys.modules["lietorch"] = lt
        sys.modules["torch_scatter"] = types.ModuleType("torch_scatter")
        with pytest.raises(ImportError, match="a different `torch_scatter` module is already imported"):
            droid_slam_b200.install_dependencies()


def _spawn(target, arg):
    """target(arg, queue, None) in a spawned process -> (exit code, what it put in the queue)"""
    ctx = multiprocessing.get_context("spawn")
    q = ctx.Queue()
    proc = ctx.Process(target=target, args=(arg, q, None))
    try:
        proc.start()
        out = q.get(timeout=300)
        proc.join(timeout=60)
    finally:
        if proc.is_alive():
            proc.terminate()
        proc.join(timeout=30)
    return proc.exitcode, out


def test_a_spawned_child_registers_the_packages_before_unpickling_its_arguments():
    """DroidAsync starts backend_process(args, video1, video2) with spawn; unpickling the DepthVideo arguments imports depth_video, which
    imports lietorch at import time.  Here the argument is an object of lietorch_user (a module doing `import lietorch` at import time) and
    the child has no other lietorch on its path: it resolves to this package because the BackendProcess, pickled first, registers it"""
    with registered_state():
        try:
            droid_slam_b200.install_dependencies()
            import lietorch_user
            modules.install_async_hook(lietorch_user, strict=False)              # no backend hooks: the child runs the module's own function
            code, out = _spawn(lietorch_user.backend_process, lietorch_user.Holder())
            assert code == 0 and out == ("droid_slam_b200.lietorch", "droid_slam_b200.lietorch", "droid_slam_b200.torch_scatter"), (code, out)
        finally:
            sys.modules.pop("lietorch_user", None)


def test_torch_scatter_against_the_stand_in():
    """the known answers of tests/test_shims_cpu.py (thirdparty/pytorch_scatter/test/test_scatter.py:12-37), on both"""
    from oracle.shims import torch_scatter as shim
    src = torch.tensor([1., 3, 2, 4, 5, 6]); index = torch.tensor([0, 1, 0, 1, 1, 3])
    cases = [(src, index, -1, None, [3, 12, 0, 6], [1.5, 4, 0, 6])]
    src2 = torch.tensor([[1., 2], [5, 6], [3, 4], [7, 8], [9, 10], [11, 12]])
    cases.append((src2, index, 0, None, [[4, 6], [21, 24], [0, 0], [11, 12]], [[2, 3], [7, 8], [0, 0], [11, 12]]))
    src3 = torch.tensor([[1., 5, 3, 7, 9, 11], [2, 4, 8, 6, 10, 12]])
    index3 = torch.tensor([[0, 1, 0, 1, 1, 3], [0, 0, 1, 0, 1, 2]])
    cases.append((src3, index3, 1, None, [[4, 21, 0, 11], [12, 18, 12, 0]], None))
    for s, i, d, n, want_sum, want_mean in cases:
        assert ts.scatter_sum(s, i, dim=d).tolist() == want_sum == shim.scatter_sum(s, i, dim=d).tolist()
        if want_mean is not None:
            assert ts.scatter_mean(s, i, dim=d).tolist() == want_mean == shim.scatter_mean(s, i, dim=d).tolist()
    assert ts.scatter_sum(torch.ones(1, 4, 2), torch.tensor([0, 0, 2, 2]), dim=1, dim_size=5).shape == (1, 5, 2)
    x = torch.randn(2, 7, 3)
    i = torch.tensor([0, 2, 2, 1, 0, 4, 4])
    assert torch.equal(ts.scatter_mean(x, i, dim=1, dim_size=6), shim.scatter_mean(x, i, dim=1, dim_size=6))
