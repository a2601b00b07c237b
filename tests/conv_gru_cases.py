"""Seeded inputs and parameters of the update operator's ConvGRU(128, 128+128+64) for the golden generator and the tests, and a stand-in
module with the reference class's layers (modules/gru.py:6-17) whose forward is the oracle's restatement, for the machines without the
reference tree.  Only seeds and sizes live here; tests/golden/conv_gru.pt holds the reference's outputs and gradients."""
import torch
import torch.nn as nn

from droid_slam_b200.modules import CONV_GRU_PARAMS
from oracle.update import conv_gru_forward

INPUT_CHANNELS = (128, 128, 64)          # inp, corr, flow


class ConvGRU(nn.Module):
    """the layers of modules/gru.py ConvGRU(h_planes, i_planes); forward = oracle.update.conv_gru_forward on them"""

    def __init__(self, h_planes=128, i_planes=320):
        super().__init__()
        self.convz = nn.Conv2d(h_planes + i_planes, h_planes, 3, padding=1)
        self.convr = nn.Conv2d(h_planes + i_planes, h_planes, 3, padding=1)
        self.convq = nn.Conv2d(h_planes + i_planes, h_planes, 3, padding=1)
        self.w = nn.Conv2d(h_planes, h_planes, 1, padding=0)
        self.convz_glo = nn.Conv2d(h_planes, h_planes, 1, padding=0)
        self.convr_glo = nn.Conv2d(h_planes, h_planes, 1, padding=0)
        self.convq_glo = nn.Conv2d(h_planes, h_planes, 1, padding=0)

    def forward(self, net, *inputs):
        return conv_gru_forward(dict(self.named_parameters()), net, *inputs, prefix="")


def make_params(seed):
    """{name: fp64 tensor} of the 14 parameters: uniform in +-1/sqrt(fan_in), as nn.Conv2d initialises them"""
    g = torch.Generator().manual_seed(seed)
    shapes = dict(convz=(128, 448, 3, 3), convr=(128, 448, 3, 3), convq=(128, 448, 3, 3), w=(128, 128, 1, 1), convz_glo=(128, 128, 1, 1),
                  convr_glo=(128, 128, 1, 1), convq_glo=(128, 128, 1, 1))
    out = {}
    for name in CONV_GRU_PARAMS:
        conv, kind = name.split(".")
        shape = shapes[conv]
        bound = (shape[1] * shape[2] * shape[3]) ** -0.5
        out[name] = (torch.rand(shape if kind == "weight" else shape[:1], generator=g, dtype=torch.float64) * 2 - 1) * bound
    return out


def load_params(module, params):
    with torch.no_grad():
        for name, p in module.named_parameters():
            p.copy_(params[name])
    return module


def make_inputs(b, h, w, seed):
    """net (tanh range, as UpdateModule's), inp (relu range), corr and flow (relu range, the encoders' outputs), fp64"""
    g = torch.Generator().manual_seed(seed)
    net = torch.tanh(torch.randn(b, 128, h, w, generator=g, dtype=torch.float64))
    ins = [torch.relu(torch.randn(b, c, h, w, generator=g, dtype=torch.float64)) for c in INPUT_CHANNELS]
    return net, ins


def make_cotangent(b, h, w, seed):
    return torch.randn(b, 128, h, w, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


# name -> (b, h, w, calls, seed): `calls` chained calls with net fed back, fresh inputs per call
CASES = {
    "b2_3x5": (2, 3, 5, 1, 1),
    "b1_1x1": (1, 1, 1, 1, 2),
    "chain2_b1_4x3": (1, 4, 3, 2, 3),
}


def case_inputs(name):
    """(params, net, [inputs per call], [cotangent per call]) of a fixture case, fp64"""
    b, h, w, calls, seed = CASES[name]
    net, _ = make_inputs(b, h, w, 100 * seed)
    ins = [make_inputs(b, h, w, 100 * seed + 1 + k)[1] for k in range(calls)]
    cots = [make_cotangent(b, h, w, 100 * seed + 50 + k) for k in range(calls)]
    return make_params(seed), net, ins, cots


def param_sample(name, t):
    """the part of a parameter gradient the fixture keeps: every element of the biases, every 13th of the 1x1 and every 257th of the 3x3
    weights (flattened), which meets every output channel"""
    stride = 1 if t.dim() == 1 else 13 if t.shape[-1] == 1 else 257
    return t.reshape(-1)[::stride].clone()


def run_chain(forward, params, net, ins, cots, keep=param_sample):
    """calls forward(net, *inputs) once per inputs, net fed back; loss = sum_k <cot_k, out_k>.  -> dict(outs, grad_net, grad_inputs
    [per call, per input], grad_params {name: keep(name, gradient)}) with params a {name: leaf tensor} the forward reads"""
    net = net.clone().requires_grad_(True)
    ins = [[t.clone().requires_grad_(True) for t in call] for call in ins]
    outs, h = [], net
    for call in ins:
        h = forward(h, *call)
        outs.append(h)
    loss = sum((o * c).sum() for o, c in zip(outs, cots))
    names = list(CONV_GRU_PARAMS)
    flat = [t for call in ins for t in call]
    g = torch.autograd.grad(loss, [net] + flat + [params[n] for n in names])
    gi = g[1:1 + len(flat)]
    return dict(outs=[o.detach() for o in outs], grad_net=g[0],
                grad_inputs=[list(gi[3 * k:3 * k + 3]) for k in range(len(ins))],
                grad_params={n: keep(n, x) for n, x in zip(names, g[1 + len(flat):])})
