"""Host side of the update operator (SURVEY section 8a row A6): `UpdateModule` with the reference's interface -- constructor-free,
the reference's submodule / parameter names (a DROID checkpoint's `update.*` entries load with `load_state_dict`), the reference's
call signature and return values (droid_slam/droid_net.py:78-143, droid_slam/modules/gru.py:5-32, droid_net.py:46-75) -- in front
of the hand-written tensor-core kernels of `csrc/update_op.cu` (C ABI `dba_update_forward`, include/droid_b200.h).

What happens here is plumbing only: the parameters are re-packed once per checkpoint into the kernels' weight layout
(`pack_update_weights`: [tap][N][K] f16, convolutions that share an input concatenated along N), `torch.unique` numbers the
aggregation segments like the reference's `GraphAgg` does, and views put the outputs into the reference's shapes.  There is NO
torch / cuDNN convolution and no CPU path: calling the module with non-CUDA tensors raises.
"""
import torch
import torch.nn as nn

__all__ = ["ConvGRU", "GraphAgg", "UpdateModule", "pack_update_weights", "PACKED_ORDER"]

# order of dba_update_weights (include/droid_b200.h)
PACKED_ORDER = ("w_corr0", "w_corr2", "w_flow0", "w_flow2", "w_gate", "w_zr", "w_q", "w_stem", "w_heads", "w_agg2", "w_eta", "w_upmask",
                "b_corr0", "b_corr2", "b_flow0", "b_flow2", "b_gate", "b_zr", "b_q", "b_stem", "b_heads", "b_agg2", "b_eta", "b_upmask",
                "w_glo", "b_glo", "b_zero")


def _conv(name):
    """parameter holder with the reference's shape for convolution `name` (table in synth.UPDATE_SHAPES); never called as a layer"""
    from .synth import UPDATE_SHAPES
    co, ci, k = UPDATE_SHAPES[name]
    return nn.Conv2d(ci, co, k, padding=k // 2)


def _taps(w, kpad=None):
    """[Co,Ci,k,k] -> [k*k (dy*k+dx), Co, Kpad] (K = input channels, zero padded)"""
    co, ci, k, _ = w.shape
    t = w.permute(2, 3, 0, 1).reshape(k * k, co, ci)
    if kpad is not None and kpad > ci:
        t = torch.cat([t, t.new_zeros(k * k, co, kpad - ci)], 2)
    return t


def _padn(t, n):
    """pad dim -2 (output channels) / a bias vector to n entries"""
    if t.dim() == 1:
        return torch.cat([t, t.new_zeros(n - t.shape[0])])
    return torch.cat([t, t.new_zeros(t.shape[0], n - t.shape[1], t.shape[2])], 1)


def pack_update_weights(sd, device=None):
    """state_dict of the update operator (reference names) -> dict of the 27 packed tensors the kernels read (layouts: droid_b200.h).
    Pure tensor re-arrangement; f16 for the tensor-core operands, f32 for biases and the global-context mat-vec."""
    f = {k: v.detach().float() for k, v in sd.items()}
    W = {}
    W["w_corr0"] = _taps(f["corr_encoder.0.weight"], 256)
    W["w_corr2"] = _taps(f["corr_encoder.2.weight"])
    w7 = f["flow_encoder.0.weight"]                                       # [128,4,7,7] -> K index (dy*7+dx)*4 + c
    W["w_flow0"] = torch.cat([w7.permute(0, 2, 3, 1).reshape(128, 196), w7.new_zeros(128, 60)], 1)[None]
    W["w_flow2"] = _taps(f["flow_encoder.2.weight"])
    W["w_gate"] = _taps(f["gru.w.weight"])
    W["w_zr"] = _taps(torch.cat([f["gru.convz.weight"], f["gru.convr.weight"]], 0))
    W["w_q"] = _taps(f["gru.convq.weight"])
    W["w_stem"] = _taps(torch.cat([f["delta.0.weight"], f["weight.0.weight"], f["agg.conv1.weight"]], 0))
    # the 3x3 / 2-channel heads as per-tap rows of one 1x1 convolution: row 4t+o = tap t of output o (delta x,y | weight x,y)
    hd = torch.zeros(1, 64, 256)
    hd[0, :36, :].view(9, 4, 256)[:, 0:2, 0:128] = _taps(f["delta.2.weight"][:2])
    hd[0, :36, :].view(9, 4, 256)[:, 2:4, 128:256] = _taps(f["weight.2.weight"][:2])
    W["w_heads"] = hd
    W["w_agg2"] = _taps(f["agg.conv2.weight"])
    we = torch.zeros(1, 32, 128)
    we[0, :9] = _taps(f["agg.eta.0.weight"])[:, 0, :]                     # row t = tap t
    W["w_eta"] = we
    W["w_upmask"] = _taps(f["agg.upmask.0.weight"])
    W["b_corr0"] = f["corr_encoder.0.bias"]; W["b_corr2"] = f["corr_encoder.2.bias"]
    W["b_flow0"] = f["flow_encoder.0.bias"]; W["b_flow2"] = f["flow_encoder.2.bias"]
    W["b_gate"] = f["gru.w.bias"]
    W["b_zr"] = torch.cat([f["gru.convz.bias"], f["gru.convr.bias"]])
    W["b_q"] = f["gru.convq.bias"]
    W["b_stem"] = torch.cat([f["delta.0.bias"], f["weight.0.bias"], f["agg.conv1.bias"]])
    W["b_heads"] = torch.cat([f["delta.2.bias"][:2], f["weight.2.bias"][:2]])
    W["b_agg2"] = f["agg.conv2.bias"]
    W["b_eta"] = f["agg.eta.0.bias"][:1]
    W["b_upmask"] = f["agg.upmask.0.bias"]
    W["w_glo"] = torch.cat([f["gru.convz_glo.weight"], f["gru.convr_glo.weight"], f["gru.convq_glo.weight"]], 0).reshape(384, 128)
    W["b_glo"] = torch.cat([f["gru.convz_glo.bias"], f["gru.convr_glo.bias"], f["gru.convq_glo.bias"]])
    W["b_zero"] = torch.zeros(64)
    out = {}
    for i, k in enumerate(PACKED_ORDER):
        t = W[k].to(torch.float16 if i < 12 else torch.float32).contiguous()
        out[k] = t.to(device) if device is not None else t
    return out


class ConvGRU(nn.Module):
    """parameters of modules/gru.py:5-17 (same names); the computation is fused into UpdateModule.forward's kernel sequence"""

    def __init__(self, prefix="gru."):
        super().__init__()
        for name in ("convz", "convr", "convq", "w", "convz_glo", "convr_glo", "convq_glo"):
            setattr(self, name, _conv(prefix + name))


class GraphAgg(nn.Module):
    """parameters of droid_net.py:46-57 (same names; GradientClip is the identity in the forward pass and has no parameters)"""

    def __init__(self, prefix="agg."):
        super().__init__()
        self.conv1, self.conv2 = _conv(prefix + "conv1"), _conv(prefix + "conv2")
        self.eta = nn.Sequential(_conv(prefix + "eta.0"), nn.Identity(), nn.Softplus())
        self.upmask = nn.Sequential(_conv(prefix + "upmask.0"))


class UpdateModule(nn.Module):
    """droid_net.py:78-143: forward(net, inp, corr, flow=None, ii=None, jj=None) -> net, delta, weight[, eta, upmask]

    Shapes as in the reference: net, inp [B,E,128,ht,wd]; corr [B,E,196,ht,wd]; flow [B,E,4,ht,wd]; returns net [B,E,128,ht,wd] (f16, a
    channels-last view: passing it back in skips the layout change), delta / weight [B,E,ht,wd,2] f32, eta [B,M',ht,wd] f32,
    upmask [B,M',576,ht,wd] f16 (M' = number of distinct source frames, ascending like torch.unique)."""

    def __init__(self):
        super().__init__()
        relu = lambda: nn.ReLU(inplace=True)
        self.corr_encoder = nn.Sequential(_conv("corr_encoder.0"), relu(), _conv("corr_encoder.2"), relu())
        self.flow_encoder = nn.Sequential(_conv("flow_encoder.0"), relu(), _conv("flow_encoder.2"), relu())
        self.weight = nn.Sequential(_conv("weight.0"), relu(), _conv("weight.2"), nn.Identity(), nn.Sigmoid())
        self.delta = nn.Sequential(_conv("delta.0"), relu(), _conv("delta.2"), nn.Identity())
        self.gru = ConvGRU()
        self.agg = GraphAgg()
        self._packed = None
        self._packed_key = None

    def packed_weights(self, device):
        from .modules import _repack_key
        key = (str(device),) + _repack_key(self.parameters())
        if self._packed is None or self._packed_key != key:
            pk = pack_update_weights(self.state_dict(), device)
            self._packed = [pk[k] for k in PACKED_ORDER]
            self._packed_key = key
        return self._packed

    def forward(self, net, inp, corr, flow=None, ii=None, jj=None):
        if not net.is_cuda:
            raise RuntimeError("droid_slam_b200.UpdateModule runs on CUDA tensors only (hand-written sm_90a kernels, no CPU path)")
        batch = net.shape[0]
        seg, n_src = None, 0
        if ii is not None:
            uniq, seg = torch.unique(ii.to(net.device), return_inverse=True)                # like GraphAgg.forward, droid_net.py:61
            if batch > 1:
                seg = (seg[None] + uniq.numel() * torch.arange(batch, device=seg.device)[:, None]).reshape(-1)
            n_src = int(uniq.numel()) * batch
        return self.forward_segments(net, inp, corr, flow, seg, n_src)

    def forward_segments(self, net, inp, corr, flow, seg, n_src):
        """forward() with GraphAgg's segments given instead of ii: seg [B*E] int64 on the device = rank of each edge's source frame
        among the distinct ones (batch b's ranks offset by b * M), n_src = B * M; seg None: no aggregation (net, delta, weight only)."""
        from . import install
        be = install()
        batch, num, ch, ht, wd = net.shape
        E = batch * num
        if _is_channels_last(net) and net.dtype == torch.float16:
            net_arg, cl = net.permute(0, 1, 3, 4, 2).reshape(E, ht, wd, ch), True         # zero-copy: already [E,ht,wd,128] in memory
        else:
            net_arg, cl = net.reshape(E, ch, ht, wd).contiguous(), False
        inp_arg = inp.reshape(E, -1, ht, wd).contiguous()
        corr_arg = corr.reshape(E, -1, ht, wd).contiguous()
        flow_arg = None if flow is None else flow.reshape(E, -1, ht, wd)
        out = be.update_forward(net_arg, inp_arg, corr_arg, flow_arg, seg, n_src, self.packed_weights(net.device), cl)
        net_new = out[0].view(batch, num, ht, wd, 128).permute(0, 1, 4, 2, 3)
        delta = out[1].view(batch, num, ht, wd, 2)
        weight = out[2].view(batch, num, ht, wd, 2)
        if seg is None:
            return net_new, delta, weight
        eta = out[3].view(batch, -1, ht, wd)
        upmask = out[4].view(batch, -1, 8 * 8 * 9, ht, wd)
        return net_new, delta, weight, eta, upmask


def _is_channels_last(t):
    """[B,E,C,H,W] tensor whose memory is [B,E,H,W,C] contiguous"""
    if t.dim() != 5:
        return False
    return t.permute(0, 1, 3, 4, 2).is_contiguous()
