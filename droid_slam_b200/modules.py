"""Hooks that put the B200-native extras under the reference's own Python classes.

The reference's `droid_slam/modules/corr.py` runs UNCHANGED on this package's `droid_backends` (its four correlation ops are the nine
drop-in callables); nothing of it is restated here.  What the reference computes in Python around those ops and this package has a
kernel for is offered as a hook:

  * `install_corr_volume_hook(corr_module)`: `CorrBlock.__init__` (modules/corr.py:24-38, 63-71: torch.matmul + 3x avg_pool2d) builds
    its four pyramid levels with the one-pass wgmma kernel `droid_backends.corr_volume_pyramid` instead.  Only the constructor is
    replaced; lookups, `cat` and `__getitem__` stay the reference's code.
  * `install_alt_corr_hook(corr_module)`: `AltCorrBlock` (modules/corr.py:89-117, the on-the-fly path of `FactorGraph.update_lowmem`
    and of the global-BA backends) on a private channels-last pyramid: `__init__` builds all levels in one launch
    (`droid_backends.altcorr_pyramid`, instead of 3x avg_pool2d) and `__call__` does every level's lookup in one launch
    (`droid_backends.altcorr_lookup_pyramid`, instead of 4x altcorr_forward + stack).  Bit-identical to the reference's call sequence;
    forward only.  The private level 0 is a copy: the block holds about 1.33x the feature maps (the reference: 0.33x extra).
  * `install_encoder_hook(extractor_module)`: `BasicEncoder.forward` (modules/extractor.py:183-198) of DroidNet's fnet (instance norm)
    and cnet (no norm) on the kernels of csrc/encoder.cu (`droid_backends.encoder_forward`) instead of cuDNN convolutions and ATen norms.
  * `reproject(...)`: `DepthVideo.reproject` (depth_video.py:171-179 -> geom/projective_ops.py:165-198) as one kernel.
  * `add_proximity_factors(graph, ...)` / `install_proximity_hook(FactorGraph)`: the edge selection of
    `FactorGraph.add_proximity_factors` (factor_graph.py:346-412) on the device (row F1).
"""
import torch

from . import install

__all__ = ["install_corr_volume_hook", "install_alt_corr_hook", "install_encoder_hook", "reproject", "upsample", "add_proximity_factors", "install_proximity_hook"]


def _corr_volume_unsupported(be, fmap1, fmap2, num_levels):
    """why corr_volume_pyramid has no kernel for these CorrBlock arguments (None: it has one)"""
    if fmap1.dim() != 5 or fmap2.shape != fmap1.shape:
        return "fmap1 and fmap2 must be [B,N,C,H,W] of one shape"
    if not (fmap1.is_cuda and fmap2.is_cuda):
        return "fmaps are not on a CUDA device"
    if fmap1.dtype != torch.float16 or fmap2.dtype != torch.float16:
        return "dtype %s / %s (float16 has a kernel)" % (fmap1.dtype, fmap2.dtype)
    if num_levels != 4:
        return "%d levels (4 has a kernel)" % num_levels
    batch, num, dim, ht, wd = fmap1.shape
    if dim != 128:
        return "%d channels (128 has a kernel)" % dim
    if ht < 8 or wd < 8:
        return "%dx%d feature maps (ht and wd must be at least 8)" % (ht, wd)
    if not be.corr_volume_supported(dim, ht, wd):
        return "no kernel for %dx%d" % (ht, wd)
    return None


def install_corr_volume_hook(corr_module, strict=True, fused_lookup=False):
    """corr_module = the imported reference module `modules.corr`.  `CorrBlock.__init__` builds its pyramid with corr_volume_pyramid for
    f16 feature maps with 128 channels, 4 levels and ht, wd >= 8.  strict: anything else raises (naming the reason) instead of silently
    taking the reference's library path; with strict=False the reference's own methods run for it.
    fused_lookup: additionally replace `CorrBlock.__call__` by the one-launch 4-level lookup `corr_lookup_pyramid`.  Where
    corr_volume_pyramid has a tiled builder (wd = 64, ht % 8 == 0) the volumes of levels 0 and 1 are kept in the tiled private layout
    (64-byte DRAM atoms, about a third less HBM traffic per lookup); elsewhere the reference layout.  Same tensor shapes, `cat` /
    `__getitem__` over edges keep working, results bit-identical to the reference-layout path."""
    be = install()
    ref_init, ref_call = corr_module.CorrBlock.__init__, corr_module.CorrBlock.__call__

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        why = _corr_volume_unsupported(be, fmap1, fmap2, num_levels)
        self._b200_native = why is None
        if why is not None:
            if strict:
                raise RuntimeError("corr_volume_pyramid has no kernel for CorrBlock(%s %s, num_levels=%d): %s"
                                   % (tuple(fmap1.shape), fmap1.dtype, num_levels, why))
            return ref_init(self, fmap1, fmap2, num_levels, radius)
        batch, num, dim, ht, wd = fmap1.shape
        tiled = bool(fused_lookup) and be.corr_volume_supported(dim, ht, wd, tiled=True)
        self.num_levels, self.radius = num_levels, radius
        idx = torch.arange(batch * num, device=fmap1.device)
        self.corr_pyramid = be.corr_volume_pyramid(fmap1.reshape(batch * num, dim, ht, wd).contiguous(), fmap2.reshape(batch * num, dim, ht, wd).contiguous(), idx, idx, tiled)
        self._b200_tiled = tiled

    def __call__(self, coords):
        if not getattr(self, "_b200_native", False):
            return ref_call(self, coords)
        batch, num, ht, wd, _ = coords.shape
        c = coords.permute(0, 1, 4, 2, 3).contiguous().view(batch * num, 2, ht, wd)
        return be.corr_lookup_pyramid([v.contiguous() for v in self.corr_pyramid], c, self._b200_tiled).view(batch, num, -1, ht, wd)

    corr_module.CorrBlock.__init__ = __init__
    if fused_lookup:
        corr_module.CorrBlock.__call__ = __call__
    return corr_module


def _alt_unsupported(fmaps, num_levels, radius):
    """why altcorr_pyramid / altcorr_lookup_pyramid have no kernel for these AltCorrBlock arguments (None: they have one)"""
    if fmaps.dim() != 5:
        return "fmaps must be [B,N,C,H,W]"
    if not fmaps.is_cuda:
        return "fmaps are not on a CUDA device"
    if fmaps.dtype not in (torch.float16, torch.float32):
        return "dtype %s (float16 and float32 have kernels)" % fmaps.dtype
    B, N, C, H, W = fmaps.shape
    if radius != 3:
        return "radius %d (3 has a kernel)" % radius
    if not 1 <= num_levels <= 4:
        return "%d levels (1..4 have kernels)" % num_levels
    if C % 8:
        return "%d channels (a multiple of 8 is needed)" % C
    if min(H, W) < 2 ** (num_levels - 1):
        return "%dx%d feature maps are too small for %d levels" % (H, W, num_levels)
    return None


def install_alt_corr_hook(corr_module, strict=True):
    """corr_module = the imported reference module `modules.corr`.  Replaces `AltCorrBlock.__init__(fmaps, num_levels=4, radius=3)` and
    `__call__(coords [B,M,H,W,2], ii, jj)` in place on the class (so `from modules.corr import AltCorrBlock` elsewhere picks it up) by
    the one-launch pyramid build and the one-launch all-level lookup on a private channels-last pyramid; the output equals the reference's
    bit for bit.  strict: fmaps / radii without a kernel (not f16/f32 on CUDA, C % 8 != 0, radius != 3, more than 4 levels) raise; with
    strict=False the reference's own methods run for them.  Forward only: inputs that require grad under grad mode raise (the hook would
    otherwise drop their gradients)."""
    be = install()
    cls = corr_module.AltCorrBlock
    ref_init, ref_call = cls.__init__, cls.__call__

    def _no_grad_inputs(*ts):
        if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in ts):
            raise RuntimeError("the native AltCorrBlock is forward only: an input requires grad")

    def __init__(self, fmaps, num_levels=4, radius=3):
        _no_grad_inputs(fmaps)
        why = _alt_unsupported(fmaps, num_levels, radius)
        if why is not None:
            if strict:
                raise RuntimeError("altcorr_pyramid has no kernel for AltCorrBlock(%s %s, num_levels=%d, radius=%d): %s"
                                   % (tuple(fmaps.shape), fmaps.dtype, num_levels, radius, why))
            self._b200_pyramid = None
            return ref_init(self, fmaps, num_levels, radius)
        self.num_levels, self.radius = num_levels, radius
        self._b200_pyramid = be.altcorr_pyramid(fmaps.contiguous(), num_levels)

    def __call__(self, coords, ii, jj):
        pyramid = getattr(self, "_b200_pyramid", None)
        if pyramid is None:
            return ref_call(self, coords, ii, jj)
        _no_grad_inputs(coords)
        if not (coords.is_cuda and coords.dtype == torch.float32 and coords.dim() == 5 and coords.shape[-1] == 2):
            raise RuntimeError("AltCorrBlock: coords must be a float32 CUDA tensor [B,M,H,W,2], got %s %s on %s"
                               % (tuple(coords.shape), coords.dtype, coords.device))
        c = coords.permute(0, 1, 4, 2, 3).contiguous()
        return be.altcorr_lookup_pyramid(pyramid, c, ii, jj, self.radius)

    cls.__init__ = __init__
    cls.__call__ = __call__
    return corr_module


def _encoder_unsupported(enc, x):
    """why encoder_forward has no kernel for this BasicEncoder and input (None: it has one)"""
    if enc.norm_fn not in ("instance", "none"):
        return "norm_fn %r (instance and none have kernels)" % (enc.norm_fn,)
    if enc.multidim:
        return "multidim"
    if getattr(enc, "dropout", None) is not None:
        return "dropout"
    if enc.conv2.out_channels not in (128, 256):
        return "output_dim %d (128 and 256 have kernels)" % enc.conv2.out_channels
    if x.dim() != 5 or x.shape[2] != 3:
        return "input must be [b,n,3,H,W]"
    if not x.is_cuda:
        return "input is not on a CUDA device"
    if x.dtype not in (torch.float16, torch.float32):
        return "dtype %s (float16 and float32 have kernels)" % x.dtype
    if x.shape[3] % 8 or x.shape[4] % 8:
        return "%dx%d images (H and W must be multiples of 8)" % (x.shape[3], x.shape[4])
    return None


def install_encoder_hook(extractor_module, strict=True):
    """extractor_module = the imported reference module `modules.extractor`.  Replaces `BasicEncoder.forward(x [b,n,3,H,W])` in place on
    the class (so droid_net.py, motion_filter.py and trajectory_filler.py pick it up unchanged) by one `encoder_forward` call: the
    module keeps the reference's parameters (a DROID checkpoint loads as before); they are packed once and re-packed when a parameter's
    storage or version changes.  Output [b,n,output_dim,H/8,W/8]: f16 under CUDA autocast (as the reference's last convolution gives),
    otherwise the input's dtype.  strict: encoders and inputs without a kernel (norm_fn other than instance / none, multidim, dropout,
    output_dim other than 128 / 256, inputs not f16/f32 on CUDA, H or W not a multiple of 8) raise; with strict=False the reference's own
    forward runs for them.  Forward only: an input that requires grad under grad mode raises, and the parameters get no gradient."""
    be = install()
    from .encoder import pack_encoder_weights
    cls = extractor_module.BasicEncoder
    ref_forward = cls.forward

    def packed(self, device):
        key = (str(device),) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if getattr(self, "_b200_packed_key", None) != key:
            self._b200_packed = pack_encoder_weights(self.state_dict(), self.norm_fn, self.conv2.out_channels, device)
            self._b200_packed_key = key
        return self._b200_packed

    def forward(self, x):
        why = _encoder_unsupported(self, x)
        if why is not None:
            if strict:
                raise RuntimeError("encoder_forward has no kernel for BasicEncoder(norm_fn=%r) on %s %s: %s" % (self.norm_fn, tuple(x.shape), x.dtype, why))
            return ref_forward(self, x)
        if torch.is_grad_enabled() and x.requires_grad:
            raise RuntimeError("the native BasicEncoder is forward only: the input requires grad")
        b, n, c, h, w = x.shape
        out = be.encoder_forward(x.reshape(b * n, c, h, w).contiguous(), packed(self, x.device), 1 if self.norm_fn == "instance" else 0,
                                 self.conv2.out_channels)
        if not torch.is_autocast_enabled("cuda"):
            out = out.to(x.dtype)
        return out.view(b, n, -1, h // 8, w // 8)

    cls.forward = forward
    return extractor_module


def reproject(poses, disps, intrinsics, ii, jj):
    """DepthVideo.reproject (reference droid_slam/depth_video.py:171-179) in one kernel: poses [N,7], disps [N,ht,wd],
    intrinsics [N,4], ii/jj index tensors or lists -> (coords [1,E,ht,wd,2], valid [1,E,ht,wd,1]) like the reference."""
    be = install()
    ii = torch.as_tensor(ii).to(device=poses.device, dtype=torch.long).reshape(-1)
    jj = torch.as_tensor(jj).to(device=poses.device, dtype=torch.long).reshape(-1)
    coords, valid = be.reproject(poses.contiguous(), disps.contiguous(), intrinsics.contiguous(), ii, jj)
    return coords[None], valid[None]


def upsample(disps, disps_up, ix, mask):
    """DepthVideo.upsample (reference droid_slam/depth_video.py:155-159) in one kernel: disps_up[ix] = cvx_upsample(disps[ix], mask).
    disps [N,ht,wd] f32, disps_up [N,8ht,8wd] f32 (written in place), ix index tensor, mask [1,len(ix),576,ht,wd] (the update operator's upmask)."""
    be = install()
    m = mask.reshape(-1, 576, disps.shape[1], disps.shape[2]).contiguous()
    disps_up[ix] = be.cvx_upsample(disps[ix].contiguous(), m)
    return disps_up


def add_proximity_factors(graph, t0=0, t1=0, rad=2, nms=2, beta=0.25, thresh=16.0, remove=False):
    """FactorGraph.add_proximity_factors (reference factor_graph.py:346-412) with the edge selection on the device (row F1).

    Same signature and effect as the reference method, `graph` being the reference's FactorGraph instance: the distance matrix stays on the
    GPU (`video.distance` -> droid_backends.frame_distance), masking / suppression / greedy selection run in
    `droid_backends.proximity_edges` (csrc/proximity.cu) instead of the Python triple loop over a CPU copy, and the resulting edge list
    -- identical, order included -- goes to the graph's own `add_factors`.  One host read (the number of edges) instead of the
    reference's `.cpu()` round trips."""
    be = install()
    video = graph.video
    t = video.counter.value
    dev = graph.ii.device
    ix = torch.arange(t0, t, device=dev)
    jx = torch.arange(t1, t, device=dev)
    ii, jj = torch.meshgrid(ix, jx, indexing="ij")
    d = video.distance(ii.reshape(-1), jj.reshape(-1), beta=beta).float().contiguous()
    ii1 = torch.cat([graph.ii, graph.ii_bad, graph.ii_inac], 0).to(torch.long).contiguous()
    jj1 = torch.cat([graph.jj, graph.jj_bad, graph.jj_inac], 0).to(torch.long).contiguous()
    es = be.proximity_edges(d, int(t0), int(t1), int(t), ii1, jj1, int(rad), int(nms), float(thresh), int(graph.max_factors), bool(video.stereo))
    graph.add_factors(es[:, 0].contiguous(), es[:, 1].contiguous(), remove)


def install_proximity_hook(factor_graph_class):
    """replace `add_proximity_factors` of the reference's FactorGraph class (factor_graph.py:346) by the device version"""
    factor_graph_class.add_proximity_factors = add_proximity_factors
    return factor_graph_class
