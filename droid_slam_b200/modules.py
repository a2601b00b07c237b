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
  * `update(graph, ...)` / `update_lowmem(graph, ...)` / `install_factor_graph_hook(FactorGraph)`: the glue of `FactorGraph.update` and
    `update_lowmem` (factor_graph.py:214-330) planned with one host read per call, every step without a host synchronisation: fused
    motion features (`droid_backends.motion_features`), the update operator on whole source frames, the write-back of its outputs
    into the graph and BA's inputs (`droid_backends.graph_writeback`).
  * `install_depth_video_hook(DepthVideo)`: `DepthVideo.reproject` / `DepthVideo.upsample` on `reproject` / `upsample` below.
"""
import sys

import torch

from . import install

__all__ = ["install_corr_volume_hook", "install_alt_corr_hook", "install_encoder_hook", "reproject", "upsample", "add_proximity_factors", "install_proximity_hook",
           "install_depth_video_hook", "update", "update_lowmem", "install_factor_graph_hook", "plan_lowmem_chunks"]


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


def install_depth_video_hook(depth_video_class):
    """replace `DepthVideo.reproject` (depth_video.py:171-179) and `DepthVideo.upsample` (:155-159) by `reproject` / `upsample` above, so
    that `FactorGraph.add_factors` takes its initial targets from the kernel the update hooks reproject with"""
    def _reproject(self, ii, jj):
        return reproject(self.poses, self.disps, self.intrinsics, ii, jj)

    def _upsample(self, ix, mask):
        upsample(self.disps, self.disps_up, ix, mask)

    depth_video_class.reproject = _reproject
    depth_video_class.upsample = _upsample
    return depth_video_class


# ---- FactorGraph.update / update_lowmem ----------------------------------------------------------------------------------------------

_LOWMEM_CHUNK_FRAMES = 8      # the reference's chunk of source frames (factor_graph.py:284); decides which edges a step updates


def _factor_graph_unsupported(graph):
    """why the update hooks cannot run this graph natively (None: they can)"""
    from .update import UpdateModule
    if not isinstance(graph.update_op, UpdateModule):
        return "graph.update_op is %s, not droid_slam_b200.update.UpdateModule" % type(graph.update_op).__name__
    video = graph.video
    for name, t in (("graph.ii", graph.ii), ("graph.net", graph.net), ("graph.target", graph.target), ("graph.damping", graph.damping),
                    ("video.poses", video.poses), ("video.disps", video.disps), ("video.intrinsics", video.intrinsics)):
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            return "%s is not a CUDA tensor" % name
    if graph.ii.numel() == 0:
        return "the graph has no edges"
    return None


def _check_native(graph):
    why = _factor_graph_unsupported(graph)
    if why is not None:
        raise RuntimeError("the native FactorGraph update cannot run this graph: %s" % why)


def _to_device(dev, arrays):
    """several CPU int64 tensors -> device views, in one pinned, non-blocking copy (no host synchronisation)"""
    sizes = [a.numel() for a in arrays]
    flat = torch.cat([a.reshape(-1).long() for a in arrays]).pin_memory().to(dev, non_blocking=True)
    return list(torch.split(flat, sizes))


def _segments(ii):
    """ascending distinct source frames of ii and each edge's rank among them (GraphAgg's torch.unique, droid_net.py:61)"""
    return torch.unique(ii, return_inverse=True)


def _corr_features(be, corr, coords, coords_t, ii=None, jj=None):
    """the graph's corr block looked up at coords [n,ht,wd,2] (coords_t: the same as [n,2,ht,wd]) -> [1,n,196,ht,wd].  A native block
    (CorrBlock under install_corr_volume_hook, AltCorrBlock under install_alt_corr_hook) goes straight to its one-launch lookup on
    coords_t; any other block is called through its own __call__."""
    n, ht, wd, _ = coords.shape
    if ii is None:
        if getattr(corr, "_b200_native", False):
            pyr = [v.contiguous() for v in corr.corr_pyramid]
            return be.corr_lookup_pyramid(pyr, coords_t, corr._b200_tiled).view(1, n, -1, ht, wd)
        return corr(coords[None])
    pyramid = getattr(corr, "_b200_pyramid", None)
    if pyramid is not None:
        return be.altcorr_lookup_pyramid(pyramid, coords_t[None], ii, jj, corr.radius)
    return corr(coords[None], ii, jj)


def update(graph, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
    """FactorGraph.update (reference factor_graph.py:214-263) with the same signature and effects, `graph` being the reference's FactorGraph
    (or an object with its attributes).  One host read plans the call (t0, the inactive edges BA uses, the source frames, BA's window);
    the motion features are one launch, the update operator one call without torch.unique, the write-back of target / weight / damping
    and BA's inputs one launch; then `video.ba` and `video.upsample` as in the reference.  Raises when the graph cannot run natively."""
    _check_native(graph)
    be = install()
    video = graph.video
    dev = graph.ii.device
    ht, wd = graph.coords0.shape[:2]
    E = graph.ii.numel()
    n_inac_all = graph.ii_inac.numel() if use_inactive else 0
    host = torch.cat([graph.ii, graph.jj] + ([graph.ii_inac, graph.jj_inac] if use_inactive else [])).long().cpu()   # the one host read
    ii, jj = host[:E], host[E:2 * E]
    if t0 is None:
        t0 = max(1, int(ii.min()) + 1)
    inac = torch.zeros(0, dtype=torch.long)
    if use_inactive:
        ii_inac, jj_inac = host[2 * E:2 * E + n_inac_all], host[2 * E + n_inac_all:]
        inac = torch.nonzero((ii_inac >= t0 - 3) & (jj_inac >= t0 - 3))[:, 0]
        ii_ba, jj_ba = torch.cat([ii_inac[inac], ii]), torch.cat([jj_inac[inac], jj])
    else:
        ii_ba, jj_ba = ii, jj
    if t1 is None:                               # what DepthVideo.ba computes with a host read of its own
        t1 = max(int(ii_ba.max()), int(jj_ba.max())) + 1
    src, seg = _segments(ii)
    seg_d, src_d, ba_frames_d, inac_d, ii_ba_d, jj_ba_d = _to_device(dev, [seg, src, torch.unique(ii_ba), inac, ii_ba, jj_ba])
    n_inac = inac.numel()

    with torch.autocast("cuda", enabled=False):
        coords, coords_t, motn = be.motion_features(video.poses, video.disps, video.intrinsics, graph.ii, graph.jj, graph.target)
        with torch.autocast("cuda", enabled=True):
            corr = _corr_features(be, graph.corr, coords, coords_t)
        graph.net, delta, weight, eta, upmask = graph.update_op.forward_segments(graph.net, graph.inp, corr, motn[None], seg_d, src.numel())
        target, weight_out = torch.empty_like(graph.target), torch.empty_like(graph.target)
        ba_target = torch.empty(n_inac + E, 2, ht, wd, device=dev)
        ba_weight = torch.empty_like(ba_target)
        if n_inac:
            ba_target[:n_inac] = graph.target_inac[0, inac_d].permute(0, 3, 1, 2)
            ba_weight[:n_inac] = graph.weight_inac[0, inac_d].permute(0, 3, 1, 2)
        damping = torch.empty(ba_frames_d.numel(), ht, wd, device=dev)
        be.graph_writeback(delta.reshape(E, ht, wd, 2), weight.reshape(E, ht, wd, 2), coords, None, target, weight_out, ba_target, ba_weight,
                           n_inac, eta[0], src_d, graph.damping, ba_frames_d, damping, EP)
        graph.target, graph.weight = target, weight_out
        video.ba(ba_target, ba_weight, damping, ii_ba_d, jj_ba_d, t0, t1, itrs=itrs, lm=1e-4, ep=0.1, motion_only=motion_only)
        if graph.upsample:
            video.upsample(src_d, upmask)
    graph.age += 1


def _lowmem_edge_budget(be, ht, wd, device):
    """the most edges one update-operator call of update_lowmem takes: a quarter of the free device memory over what one edge needs
    (its share of the operator's workspace with every edge its own source frame, its corr features and the operator's outputs)"""
    hw = ht * wd
    per_edge = -(-be.update_workspace_bytes(64, 64, ht, wd) // 64) + hw * (196 * 2 + 128 * 2 + 2 * 2 * 4 + 4 + 576 * 2)
    free, _ = torch.cuda.mem_get_info(device)
    return max(1, (free // 4) // per_edge)


def plan_lowmem_chunks(ii, jj, max_edges):
    """Plan of one update_lowmem step over the graph edges ii, jj (CPU int64).

    The edges the reference updates are those whose source frame falls in one of its chunks range(ii.min(), jj.max() + 1, 8) of 8 source
    frames.  They are cut into chunks of whole source frames (ascending) holding at most max_edges edges, except a single source frame
    with more edges, which is a chunk of its own.  GraphAgg averages over the edges of one source frame only, so any such cut computes
    what the reference's chunks compute.
    Returns (perm, chunks, src, seg): perm [n] graph edge ids in call order (chunk by chunk, graph order inside a chunk); chunks a list of
    (row_lo, row_hi, src_lo, src_hi); src the ascending source frames of each chunk, concatenated; seg [n] each row's rank among its
    chunk's source frames."""
    ii, jj = ii.long(), jj.long()
    first = int(ii.min())
    n_ref = len(range(first, int(jj.max()) + 1, _LOWMEM_CHUNK_FRAMES))
    covered = ii < first + _LOWMEM_CHUNK_FRAMES * n_ref
    frames, counts = torch.unique(ii[covered], return_counts=True)
    chunk_of_frame, frame_lo, acc = [], [], 0
    for k, c in enumerate(counts.tolist()):
        if not frame_lo or (acc > 0 and acc + c > max_edges):
            frame_lo.append(k)
            acc = 0
        chunk_of_frame.append(len(frame_lo) - 1)
        acc += c
    edges = torch.nonzero(covered)[:, 0]
    pos = torch.searchsorted(frames, ii[edges])
    key = torch.as_tensor(chunk_of_frame, dtype=torch.long)[pos] if edges.numel() else pos
    order = torch.sort(key, stable=True).indices
    perm, key, pos = edges[order], key[order], pos[order]
    seg = pos - torch.as_tensor(frame_lo, dtype=torch.long)[key] if edges.numel() else pos
    chunks, row = [], 0
    frame_hi = frame_lo[1:] + [frames.numel()]
    for lo, hi in zip(frame_lo, frame_hi):
        n = int(counts[lo:hi].sum())
        chunks.append((row, row + n, lo, hi))
        row += n
    return perm, chunks, frames, seg


def _alt_corr_class(graph):
    """the AltCorrBlock the graph's module imported (the reference's factor_graph.py: `from modules.corr import CorrBlock, AltCorrBlock`);
    under install_alt_corr_hook it is the native block"""
    return sys.modules[type(graph).__module__].AltCorrBlock


def update_lowmem(graph, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, steps=8):
    """FactorGraph.update_lowmem (reference factor_graph.py:266-330) with the same signature and effects.  One host read per call plans
    every step: the edges the reference's 8-frame chunks cover, cut into chunks of whole source frames sized to the free device memory,
    and BA's frame list.  The context features, the graph's net in call order and BA's inputs for the edges the operator does not touch
    are gathered once per call.  Each step: one motion_features launch, per chunk the corr lookup, the update operator and
    graph_writeback, then video.upsample (when graph.upsample) and video.ba -- no host synchronisation.  graph.net is scattered back into
    graph order at the end of the call.  Raises when the graph cannot run natively."""
    _check_native(graph)
    be = install()
    video = graph.video
    dev = graph.ii.device
    t = video.counter.value
    num, rig, ch, ht, wd = video.fmaps.shape
    E = graph.ii.numel()
    n_inac = graph.ii_inac.numel() if use_inactive else 0
    host = torch.cat([graph.ii, graph.jj] + ([graph.ii_inac] if use_inactive else [])).long().cpu()     # the one host read
    ii, jj = host[:E], host[E:2 * E]
    ii_ba = torch.cat([host[2 * E:], ii])
    perm, chunks, src, seg = plan_lowmem_chunks(ii, jj, _lowmem_edge_budget(be, ht, wd, dev))
    ip, jp = ii[perm], jj[perm]
    perm_d, seg_d, src_d, ii_alt_d, jj_alt_d, ba_frames_d = _to_device(
        dev, [perm, seg, src, rig * ip, rig * jp + (ip == jp).long(), torch.unique(ii_ba)])

    with torch.autocast("cuda", enabled=False):
        corr_op = _alt_corr_class(graph)(video.fmaps.view(1, num * rig, ch, ht, wd))
        inp = video.inps[graph.ii[perm_d]]
        if graph.net.dtype == torch.float16:     # channels-last: the update operator reads it without a layout change
            net = torch.empty(perm.numel(), ht, wd, graph.net.shape[2], dtype=graph.net.dtype, device=dev).permute(0, 3, 1, 2)
        else:
            net = torch.empty(perm.numel(), *graph.net.shape[2:], dtype=graph.net.dtype, device=dev)
        net.copy_(graph.net[0, perm_d])
        if use_inactive:
            ii_ba_d, jj_ba_d = torch.cat([graph.ii_inac, graph.ii]), torch.cat([graph.jj_inac, graph.jj])
            ba_target = torch.cat([graph.target_inac[0], graph.target[0]]).permute(0, 3, 1, 2).contiguous()
            ba_weight = torch.cat([graph.weight_inac[0], graph.weight[0]]).permute(0, 3, 1, 2).contiguous()
        else:
            ii_ba_d, jj_ba_d = graph.ii, graph.jj
            ba_target = graph.target[0].permute(0, 3, 1, 2).contiguous()
            ba_weight = graph.weight[0].permute(0, 3, 1, 2).contiguous()
        damping = torch.empty(ba_frames_d.numel(), ht, wd, device=dev)
        no_rows = torch.empty(0, ht, wd, 2, device=dev)

        for _ in range(steps):
            if chunks:
                coords, coords_t, motn = be.motion_features(video.poses, video.disps, video.intrinsics, graph.ii, graph.jj, graph.target, perm_d)
            for c, (a, b, s0, s1) in enumerate(chunks):
                with torch.autocast("cuda", enabled=True):
                    corr = _corr_features(be, corr_op, coords[a:b], coords_t[a:b], ii_alt_d[a:b], jj_alt_d[a:b])
                    net_new, delta, weight, eta, upmask = graph.update_op.forward_segments(net[a:b][None], inp[a:b][None], corr, motn[a:b][None],
                                                                                          seg_d[a:b], s1 - s0)
                    if graph.upsample:
                        video.upsample(src_d[s0:s1], upmask)
                net[a:b] = net_new[0]
                last = c == len(chunks) - 1
                be.graph_writeback(delta[0], weight[0], coords[a:b], perm_d[a:b], graph.target, graph.weight, ba_target, ba_weight, n_inac,
                                   eta[0], src_d[s0:s1], graph.damping, ba_frames_d if last else None, damping if last else None, EP)
            if not chunks:                       # no edge in the reference's chunks: BA's damping still has to be gathered
                be.graph_writeback(no_rows, no_rows, no_rows, None, graph.target, graph.weight, ba_target, ba_weight, n_inac,
                                   None, None, graph.damping, ba_frames_d, damping, EP)
            graph.age += 1
            video.ba(ba_target, ba_weight, damping, ii_ba_d, jj_ba_d, 1, t, itrs=itrs, lm=1e-5, ep=1e-2, motion_only=False)
            video.dirty[:t] = True
        graph.net[0, perm_d] = net


def install_factor_graph_hook(factor_graph_class, strict=True):
    """replace `update` and `update_lowmem` of the reference's FactorGraph class (factor_graph.py:214, :266) by the native versions above.
    strict: a graph they cannot run (update_op not droid_slam_b200.update.UpdateModule, tensors not on CUDA, no edges) raises, naming the
    reason; with strict=False the reference's own method runs for it."""
    ref_update, ref_lowmem = factor_graph_class.update, factor_graph_class.update_lowmem

    def _update(self, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
        if not strict and _factor_graph_unsupported(self) is not None:
            return ref_update(self, t0, t1, itrs, use_inactive, EP, motion_only)
        return update(self, t0, t1, itrs, use_inactive, EP, motion_only)

    def _update_lowmem(self, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, steps=8):
        if not strict and _factor_graph_unsupported(self) is not None:
            return ref_lowmem(self, t0, t1, itrs, use_inactive, EP, steps)
        return update_lowmem(self, t0, t1, itrs, use_inactive, EP, steps)

    factor_graph_class.update = _update
    factor_graph_class.update_lowmem = _update_lowmem
    return factor_graph_class
