"""The pure-PyTorch stand-ins for lietorch / torch_scatter (oracle/shims, test infrastructure) against the identities and known
answers of the packages' own tests: thirdparty/lietorch/lietorch/run_tests.py:16-52, thirdparty/pytorch_scatter/test/test_scatter.py:12-60."""
import torch

import oracle
from oracle.shims import lietorch, torch_scatter
from oracle.shims.lietorch import SE3, SO3


def _g(seed=0):
    return torch.Generator().manual_seed(seed)


def test_exp_log():                                                 # run_tests.py:16-21
    for G in (SE3, SO3):
        a = .2 * torch.randn(2, 3, 4, 5, G.manifold_dim, generator=_g(1)).double()
        assert torch.allclose(a, G.exp(a).log(), atol=1e-8)


def test_inv():                                                     # run_tests.py:23-28
    for G in (SE3, SO3):
        X = G.exp(.1 * torch.randn(2, 3, 4, 5, G.manifold_dim, generator=_g(2)).double())
        a = (X * X.inv()).log()
        assert torch.allclose(a, torch.zeros_like(a), atol=1e-8)


def test_adj():                                                     # run_tests.py:30-41: X Exp(a) == Exp(Adj(X) a) X
    X = SE3.exp(torch.randn(2, 3, 4, 5, 6, generator=_g(3)).double())
    a = torch.randn(2, 3, 4, 5, 6, generator=_g(4)).double()
    c = ((X * SE3.exp(a)) * (SE3.exp(X.adj(a)) * X).inv()).log()
    assert torch.allclose(c, torch.zeros_like(c), atol=1e-8)
    b = torch.randn(2, 3, 4, 5, 6, generator=_g(5)).double()
    assert torch.allclose((X.adj(a) * b).sum(-1), (a * X.adjT(b)).sum(-1), atol=1e-9)     # adjT is the transpose of adj


def test_act():                                                     # run_tests.py:44-52
    X = SE3.exp(torch.randn(1, 6, generator=_g(6)).double())
    p = torch.randn(1, 3, generator=_g(7)).double()
    ph = torch.cat([p, torch.ones(1, 1).double()], -1)
    assert torch.allclose(X.act(p), (X.matrix() @ ph[..., None])[..., 0][..., :3], atol=1e-8)
    assert torch.allclose(X.act(ph)[..., :3], X.act(p), atol=1e-12)


def test_retr_and_group_product_agree_with_the_kernel_restatement():
    """the stand-in's Exp(a)*T equals the oracle's restatement of the reference's CUDA retraction (src/droid_kernels.cu:886-904) for
    unit quaternions"""
    g = _g(8)
    T = SE3.exp(torch.randn(7, 6, generator=g).double())
    a = 0.1 * torch.randn(7, 6, generator=g).double()
    t1, q1 = oracle.retr_se3(a, T.data[:, :3], T.data[:, 3:])
    R = T.retr(a).data
    assert torch.allclose(R[:, :3], t1, atol=1e-10) and torch.allclose(R[:, 3:], q1, atol=1e-10)
    tij, qij = oracle.rel_se3(T.data[:3, :3], T.data[:3, 3:], T.data[3:6, :3], T.data[3:6, 3:])
    Gij = (T[3:6] * T[:3].inv()).data
    assert torch.allclose(Gij[:, :3], tij, atol=1e-10) and torch.allclose(Gij[:, 3:], qij, atol=1e-10)


def test_identity_indexing_cat():
    I = SE3.Identity(2, 3)
    assert I.shape == (2, 3) and torch.equal(I.data[0, 0], SE3.id_elem)
    X = SE3.exp(torch.randn(1, 5, 6, generator=_g(9)))
    assert X[:, torch.tensor([0, 2])].shape == (1, 2) and X[:, :, None, None].data.shape == (1, 5, 1, 1, 7)
    assert lietorch.cat([X, X], 1).shape == (1, 10) and SE3.IdentityLike(X).shape == (1, 5)


def test_scatter_known_answers():                                   # test_scatter.py:12-37
    src = torch.tensor([1., 3, 2, 4, 5, 6]); index = torch.tensor([0, 1, 0, 1, 1, 3])
    assert torch_scatter.scatter_sum(src, index, dim=-1).tolist() == [3, 12, 0, 6]
    assert torch_scatter.scatter_mean(src, index, dim=-1).tolist() == [1.5, 4, 0, 6]
    src = torch.tensor([[1., 2], [5, 6], [3, 4], [7, 8], [9, 10], [11, 12]])
    assert torch_scatter.scatter_sum(src, index, dim=0).tolist() == [[4, 6], [21, 24], [0, 0], [11, 12]]
    assert torch_scatter.scatter_mean(src, index, dim=0).tolist() == [[2, 3], [7, 8], [0, 0], [11, 12]]
    src = torch.tensor([[1., 5, 3, 7, 9, 11], [2, 4, 8, 6, 10, 12]])
    index2 = torch.tensor([[0, 1, 0, 1, 1, 3], [0, 0, 1, 0, 1, 2]])
    assert torch_scatter.scatter_sum(src, index2, dim=1).tolist() == [[4, 21, 0, 11], [12, 18, 12, 0]]
    assert torch_scatter.scatter_sum(torch.ones(1, 4, 2), torch.tensor([0, 0, 2, 2]), dim=1, dim_size=5).shape == (1, 5, 2)
