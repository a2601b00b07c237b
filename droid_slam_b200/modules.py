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
  * `fill_trajectory(filler, stream)` / `install_trajectory_filler_hook(trajectory_filler)`: `PoseTrajectoryFiller.__call__`
    (trajectory_filler.py:42-110) with on-device pose interpolation (`droid_backends.fill_interpolate`), batches sized by free device
    memory and a one-launch motion-only BA per update (`droid_backends.pose_only_ba`).
  * `track(filter, ...)` / `install_motion_filter_hook(motion_filter)`: `MotionFilter.track` (motion_filter.py:50-91) with camera frames
    fed straight into the encoders (`droid_backends.encoder_forward_frames`), the motion probe on the correlation kernels and one host
    read per frame (row F6).

  * `install_update_module_hook(droid_net)`: DroidNet (and both reference `load_network` functions) build the native update operator.
  * `install_async_hook(droid_async)`: DroidAsync's backend process (droid_async.py:37-130), started with `spawn`, re-installs every hook
    of the parent (`hook_registry`) and runs the reference's loop with the frontend -> backend hand-over on the device
    (`handover_round` -> `droid_backends.fragment_handover`, one host sync per round).
  * `droid_slam_b200.install_dependencies()` (the package's, recorded here too): `lietorch` / `torch_scatter` resolve to the package's own,
    in the spawned backend before its arguments are unpickled (`_unpickle_backend`).
  * `install_corr_training_hook(droid_net)`: DroidNet's CorrBlock (modules/corr.py:6-71, `droid_net.CorrBlock`) on fp32 feature maps,
    forward and backward, on csrc/corr_train.cu, so `train.py`'s loss reaches fnet through native kernels.
  * `ba_layer(...)` / `install_ba_layer_hook(droid_net)`: DroidNet's differentiable dense BA (geom/ba.py:31-106, `droid_net.BA`) forward
    and backward on csrc/ba_layer.cu (`droid_backends.ba_layer_forward` / `ba_layer_backward`), so `train.py` trains through it.
  * `flow_loss(...)` / `install_flow_loss_hook(losses)`: train.py's flow loss (geom/losses.py:89-118, `losses.flow_loss`) with every
    iterate in one pass over the full-resolution pixels and its backward (`droid_backends.flow_loss_forward` / `flow_loss_backward`).
  * `upsample_disp(...)` / `install_upsample_disp_hook(droid_net)`: DroidNet's disparity upsampling (droid_net.py:37-42,
    `droid_net.upsample_disp`) on `droid_backends.cvx_upsample` with its backward (`cvx_upsample_backward`).
  * `conv_gru(module, net, *inputs)` / `install_conv_gru_hook(gru)`: the update operator's ConvGRU (modules/gru.py:19-32,
    `ConvGRU.forward`) forward and backward on csrc/gru_train.cu (`droid_backends.conv_gru_forward` / `conv_gru_backward`).

The strict policy, one for every hook with a `strict` flag (`_replace`): each call first asks, once, whether the native path can run
it.  If not, strict=True (the default) raises RuntimeError naming the replaced method or global and the reason; strict=False runs the
reference's own function -- the one the first install found, however often the hook is installed again.  `update`, `update_lowmem`,
`fill_trajectory`, `track`, `ba_layer`, `CorrBlock`, `flow_loss`, `upsample_disp` and `conv_gru` called directly raise in the same
words.
"""
import copy
import importlib
import sys
import time
import types

import torch

from . import install

__all__ = ["install_corr_volume_hook", "install_alt_corr_hook", "install_encoder_hook", "reproject", "upsample", "add_proximity_factors", "install_proximity_hook",
           "install_depth_video_hook", "update", "update_lowmem", "install_factor_graph_hook", "plan_lowmem_chunks", "fill_trajectory",
           "install_trajectory_filler_hook", "track", "install_motion_filter_hook", "hook_registry", "reinstall_hooks",
           "install_update_module_hook", "handover_round", "BackendProcess", "install_async_hook", "ba_layer", "install_ba_layer_hook",
           "install_corr_training_hook", "flow_loss", "install_flow_loss_hook", "upsample_disp", "install_upsample_disp_hook", "conv_gru",
           "install_conv_gru_hook"]


def _require(entry, why):
    """raise for a call of `entry` the native path cannot run (why: the reason; None: it can run it)"""
    if why is not None:
        raise RuntimeError("%s has no kernel for this call: %s" % (entry, why))


def _original(owner, name):
    """owner.<name> as the reference defines it: taken on the first call and kept on the owner as _b200_reference_<name>, so that a hook
    installed again reaches the reference's own function, not the previous install's replacement"""
    key = "_b200_reference_" + name
    ref = vars(owner).get(key, getattr(owner, name))
    setattr(owner, key, ref)
    return ref


def _replace(owner, name, native, unsupported, strict):
    """replace `name` of `owner` -- a method of a reference class, or a global of a reference module -- by native under the strict
    policy.  unsupported, native and the reference's own function (_original) all take the replacement's arguments, self first for a
    method; unsupported gives why the native path cannot run the call (None: it can)"""
    ref = _original(owner, name)
    entry = "%s.%s" % (owner.__name__, name) if isinstance(owner, type) else name

    def replacement(*args, **kwargs):
        why = unsupported(*args, **kwargs)
        if why is not None and not strict:
            return ref(*args, **kwargs)
        _require(entry, why)
        return native(*args, **kwargs)

    setattr(owner, name, replacement)


def _graph_unsupported(who, obj, update, encoders=(), own=(), video=()):
    """why `obj` (`who` in the reason) cannot run natively for its operators and buffers (None: it can): obj.<update> must be
    droid_slam_b200.update.UpdateModule, obj.<encoders> under install_encoder_hook, obj.<own> and obj.video.<video> CUDA tensors"""
    from .update import UpdateModule
    if not isinstance(getattr(obj, update), UpdateModule):
        return "%s.%s is %s, not droid_slam_b200.update.UpdateModule" % (who, update, type(getattr(obj, update)).__name__)
    for name in encoders:
        if not getattr(type(getattr(obj, name)).forward, "_b200_encoder_hook", False):
            return "%s.%s (%s) is not a BasicEncoder under install_encoder_hook" % (who, name, type(getattr(obj, name)).__name__)
    for prefix, owner, names in ((who, obj, own), ("video", obj.video, video)):
        for name in names:
            t = getattr(owner, name, None)
            if not (isinstance(t, torch.Tensor) and t.is_cuda):
                return "%s.%s is not a CUDA tensor" % (prefix, name)
    return None


def _repack_key(tensors):
    """(data_ptr, version) of each tensor: a cache built from them is stale once this changes (a tensor replaced or modified in place)"""
    return tuple((t.data_ptr(), t._version) for t in tensors)


def _stage(dev, *tensors):
    """tensors to the device without a host synchronisation, shapes kept.  One tensor: by pinned staging and a non-blocking copy, or
    passed through when already on the device.  Several CPU tensors of one dtype: in one such copy, as views of one buffer."""
    if len(tensors) > 1:
        flat = _stage(dev, torch.cat([t.reshape(-1) for t in tensors]))
        return [v.view(t.shape) for v, t in zip(torch.split(flat, [t.numel() for t in tensors]), tensors)]
    return tensors[0].to(dev) if tensors[0].is_cuda else tensors[0].pin_memory().to(dev, non_blocking=True)


def _update_edge_bytes(be, ht, wd):
    """one edge's share of the update operator's workspace, every edge its own source frame"""
    return -(-be.update_workspace_bytes(64, 64, ht, wd) // 64)


def _quarter_free(device, unit_bytes):
    """how many units of unit_bytes a quarter of the free device memory holds, at least 1"""
    free, _ = torch.cuda.mem_get_info(device)
    return max(1, (free // 4) // unit_bytes)


def _volumes(be, fmap1, fmap2, ii, jj, tiled=True):
    """the 4-level correlation volumes of fmap1[ii] with fmap2[jj] (f16 [.,C,ht,wd]) -> (pyramid, tiled).  tiled: take the tiled private
    layout (64-byte DRAM atoms) wherever corr_volume_pyramid has a tiled builder; otherwise, and with tiled=False, the reference layout"""
    tiled = bool(tiled) and be.corr_volume_supported(*fmap1.shape[-3:], tiled=True)
    return be.corr_volume_pyramid(fmap1, fmap2, ii, jj, tiled), tiled


def _lookup(be, pyramid, tiled, coords_t):
    """the one-launch 4-level lookup of volumes from _volumes (or CorrBlock's) at coords_t [n,2,ht,wd] -> [1,n,196,ht,wd]"""
    n, _, ht, wd = coords_t.shape
    return be.corr_lookup_pyramid([v.contiguous() for v in pyramid], coords_t, tiled).view(1, n, -1, ht, wd)


def _no_grad_inputs(who, *ts):
    """raise for a forward-only native `who` when one of ts is a tensor that requires grad under grad mode (its gradient would be dropped)"""
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in ts):
        raise RuntimeError("the native %s is forward only: an input requires grad" % who)


def _corr_fmaps_unsupported(fmap1, fmap2, num_levels):
    """why no CorrBlock kernel, of either dtype, takes these arguments (None: one may): both hooks need [B,N,128,ht,wd] CUDA feature maps
    of one shape with ht, wd >= 8, and 4 levels"""
    if fmap1.dim() != 5 or fmap2.shape != fmap1.shape:
        return "fmap1 and fmap2 must be [B,N,C,H,W] of one shape"
    if not (fmap1.is_cuda and fmap2.is_cuda):
        return "fmaps are not on a CUDA device"
    if num_levels != 4:
        return "%d levels (4 has a kernel)" % num_levels
    dim, ht, wd = fmap1.shape[2:]
    if dim != 128:
        return "%d channels (128 has a kernel)" % dim
    if ht < 8 or wd < 8:
        return "%dx%d feature maps (ht and wd must be at least 8)" % (ht, wd)
    return None


def _corr_volume_unsupported(be, fmap1, fmap2, num_levels):
    """why corr_volume_pyramid has no kernel for these CorrBlock arguments (None: it has one)"""
    why = _corr_fmaps_unsupported(fmap1, fmap2, num_levels)
    if why is not None:
        return why
    if fmap1.dtype != torch.float16 or fmap2.dtype != torch.float16:
        return "dtype %s / %s (float16 has a kernel)" % (fmap1.dtype, fmap2.dtype)
    dim, ht, wd = fmap1.shape[2:]
    if not be.corr_volume_supported(dim, ht, wd):
        return "no kernel for %dx%d" % (ht, wd)
    return None


def install_corr_volume_hook(corr_module, strict=True, fused_lookup=False):
    """corr_module = the imported reference module `modules.corr`.  `CorrBlock.__init__` builds its pyramid with corr_volume_pyramid for
    f16 feature maps with 128 channels, 4 levels and ht, wd >= 8; anything else follows the strict policy (module docstring).
    fused_lookup: additionally replace `CorrBlock.__call__` by the one-launch 4-level lookup `corr_lookup_pyramid`.  Where
    corr_volume_pyramid has a tiled builder (wd = 64, ht % 8 == 0) the volumes of levels 0 and 1 are kept in the tiled private layout
    (64-byte DRAM atoms, about a third less HBM traffic per lookup); elsewhere the reference layout.  Same tensor shapes, `cat` /
    `__getitem__` over edges keep working, results bit-identical to the reference-layout path.  Forward only: feature maps that require grad
    under grad mode raise, whichever constructor would run (install_corr_training_hook is the differentiable block)."""
    be = install()
    cls = corr_module.CorrBlock
    ref_call = _original(cls, "__call__")

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        batch, num, dim, ht, wd = fmap1.shape
        self.num_levels, self.radius = num_levels, radius
        idx = torch.arange(batch * num, device=fmap1.device)
        self.corr_pyramid, self._b200_tiled = _volumes(be, fmap1.reshape(batch * num, dim, ht, wd).contiguous(),
                                                       fmap2.reshape(batch * num, dim, ht, wd).contiguous(), idx, idx, fused_lookup)

    def __call__(self, coords):
        if self._b200_tiled is None:
            return ref_call(self, coords)
        batch, num, ht, wd, _ = coords.shape
        c = coords.permute(0, 1, 4, 2, 3).contiguous().view(batch * num, 2, ht, wd)
        return _lookup(be, self.corr_pyramid, self._b200_tiled, c).view(batch, num, -1, ht, wd)

    cls._b200_tiled = None                      # a block's volume layout (True: tiled); None where the reference's constructor ran
    def unsupported(blk, fmap1, fmap2, num_levels=4, radius=3):
        _no_grad_inputs("CorrBlock", fmap1, fmap2)   # an input check, ahead of the policy
        return _corr_volume_unsupported(be, fmap1, fmap2, num_levels)

    _replace(cls, "__init__", __init__, unsupported, strict)
    if fused_lookup:
        cls.__call__ = __call__
    _record("install_corr_volume_hook", corr_module, strict=strict, fused_lookup=fused_lookup)
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
    bit for bit.  Kernels exist for f16/f32 fmaps on CUDA with C % 8 == 0, radius 3 and 1-4 levels; anything else follows the strict
    policy (module docstring).  Forward only: inputs that require grad under grad mode raise, whichever constructor would run (the hook
    would otherwise drop their gradients)."""
    be = install()
    cls = corr_module.AltCorrBlock
    ref_call = _original(cls, "__call__")

    def __init__(self, fmaps, num_levels=4, radius=3):
        self.num_levels, self.radius = num_levels, radius
        self._b200_pyramid = be.altcorr_pyramid(fmaps.contiguous(), num_levels)

    def unsupported(self, fmaps, num_levels=4, radius=3):
        _no_grad_inputs("AltCorrBlock", fmaps)   # an input check, ahead of the policy
        return _alt_unsupported(fmaps, num_levels, radius)

    def __call__(self, coords, ii, jj):
        if self._b200_pyramid is None:
            return ref_call(self, coords, ii, jj)
        _no_grad_inputs("AltCorrBlock", coords)
        if not (coords.is_cuda and coords.dtype == torch.float32 and coords.dim() == 5 and coords.shape[-1] == 2):
            raise RuntimeError("AltCorrBlock: coords must be a float32 CUDA tensor [B,M,H,W,2], got %s %s on %s"
                               % (tuple(coords.shape), coords.dtype, coords.device))
        c = coords.permute(0, 1, 4, 2, 3).contiguous()
        return be.altcorr_lookup_pyramid(self._b200_pyramid, c, ii, jj, self.radius)

    cls._b200_pyramid = None                    # a block's private pyramid; None where the reference's constructor ran
    _replace(cls, "__init__", __init__, unsupported, strict)
    cls.__call__ = __call__
    _record("install_alt_corr_hook", corr_module, strict=strict)
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
    otherwise the input's dtype.  Kernels exist for norm_fn instance / none, no multidim, no dropout, output_dim 128 / 256 and f16/f32
    inputs on CUDA with H and W multiples of 8; anything else follows the strict policy (module docstring).  Forward only: an input that
    requires grad under grad mode raises, and the parameters get no gradient."""
    be = install()

    def forward(self, x):
        _no_grad_inputs("BasicEncoder", x)
        b, n, c, h, w = x.shape
        out = be.encoder_forward(x.reshape(b * n, c, h, w).contiguous(), _packed_encoder(self, x.device), 1 if self.norm_fn == "instance" else 0,
                                 self.conv2.out_channels)
        if not torch.is_autocast_enabled("cuda"):
            out = out.to(x.dtype)
        return out.view(b, n, -1, h // 8, w // 8)

    _replace(extractor_module.BasicEncoder, "forward", forward, lambda enc, x: _encoder_unsupported(enc, x), strict)
    extractor_module.BasicEncoder.forward._b200_encoder_hook = True          # what the filler and motion-filter checks look for
    _record("install_encoder_hook", extractor_module, strict=strict)
    return extractor_module


def _packed_encoder(enc, device):
    """the BasicEncoder's parameters in the kernels' layout, packed once and re-packed when a parameter's storage or version changes"""
    from .encoder import pack_encoder_weights
    key = (str(device),) + _repack_key(enc.parameters())
    if getattr(enc, "_b200_packed_key", None) != key:
        enc._b200_packed = pack_encoder_weights(enc.state_dict(), enc.norm_fn, enc.conv2.out_channels, device)
        enc._b200_packed_key = key
    return enc._b200_packed


def _frame_norm(owner):
    """owner.MEAN / owner.STDV (the reference's [3,1,1] normalisation constants, possibly on the device) as two lists of 3 floats; read
    from the device once and again only when either tensor is replaced or modified"""
    key = _repack_key((owner.MEAN, owner.STDV))
    cached = getattr(owner, "_b200_frame_norm", None)
    if cached is None or cached[0] != key:
        cached = (key, owner.MEAN.reshape(-1).tolist(), owner.STDV.reshape(-1).tolist())
        owner._b200_frame_norm = cached
    return cached[1], cached[2]


def _encode_frames(be, enc, frames, norm):
    """a BasicEncoder under install_encoder_hook on uint8 BGR camera frames [n,3,H,W] on the device -> [n,output_dim,H/8,W/8] f16, with the
    reference's channel flip and normalisation (norm = _frame_norm(...)) done on load by the encoder's first kernel: the bits of the
    hooked forward under autocast on `(frames[:, [2, 1, 0]] / 255.0).sub_(MEAN).div_(STDV)`, without that fp32 copy"""
    return be.encoder_forward_frames(frames.contiguous(), _packed_encoder(enc, frames.device), 1 if enc.norm_fn == "instance" else 0,
                                     enc.conv2.out_channels, True, norm[0], norm[1])


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
    _record("install_proximity_hook", factor_graph_class)
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
    _record("install_depth_video_hook", depth_video_class)
    return depth_video_class


# ---- FactorGraph.update / update_lowmem ----------------------------------------------------------------------------------------------

_LOWMEM_CHUNK_FRAMES = 8      # the reference's chunk of source frames (factor_graph.py:284); decides which edges a step updates


def _factor_graph_unsupported(graph):
    """why the update hooks cannot run this graph natively (None: they can)"""
    why = _graph_unsupported("graph", graph, "update_op", own=("ii", "net", "target", "damping"), video=("poses", "disps", "intrinsics"))
    if why is None and graph.ii.numel() == 0:
        return "the graph has no edges"
    return why


def _segments(ii):
    """ascending distinct source frames of ii and each edge's rank among them (GraphAgg's torch.unique, droid_net.py:61)"""
    return torch.unique(ii, return_inverse=True)


def _corr_features(be, corr, coords, coords_t, ii=None, jj=None):
    """the graph's corr block looked up at coords [n,ht,wd,2] (coords_t: the same as [n,2,ht,wd]) -> [1,n,196,ht,wd].  A native block
    (CorrBlock under install_corr_volume_hook, AltCorrBlock under install_alt_corr_hook) goes straight to its one-launch lookup on
    coords_t; any other block is called through its own __call__."""
    if ii is None:
        tiled = getattr(corr, "_b200_tiled", None)
        return corr(coords[None]) if tiled is None else _lookup(be, corr.corr_pyramid, tiled, coords_t)
    pyramid = getattr(corr, "_b200_pyramid", None)
    return corr(coords[None], ii, jj) if pyramid is None else be.altcorr_lookup_pyramid(pyramid, coords_t[None], ii, jj, corr.radius)


def update(graph, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
    """FactorGraph.update (reference factor_graph.py:214-263) with the same signature and effects, `graph` being the reference's FactorGraph
    (or an object with its attributes).  One host read plans the call (t0, the inactive edges BA uses, the source frames, BA's window);
    the motion features are one launch, the update operator one call without torch.unique, the write-back of target / weight / damping
    and BA's inputs one launch; then `video.ba` and `video.upsample` as in the reference.  Raises when the graph cannot run natively."""
    _require("FactorGraph.update", _factor_graph_unsupported(graph))
    _update(graph, t0, t1, itrs, use_inactive, EP, motion_only)


def _update(graph, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
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
    seg_d, src_d, ba_frames_d, inac_d, ii_ba_d, jj_ba_d = _stage(dev, seg, src, torch.unique(ii_ba), inac, ii_ba, jj_ba)
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
    return _quarter_free(device, _update_edge_bytes(be, ht, wd) + ht * wd * (196 * 2 + 128 * 2 + 2 * 2 * 4 + 4 + 576 * 2))


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
    _require("FactorGraph.update_lowmem", _factor_graph_unsupported(graph))
    _update_lowmem(graph, t0, t1, itrs, use_inactive, EP, steps)


def _update_lowmem(graph, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, steps=8):
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
    perm_d, seg_d, src_d, ii_alt_d, jj_alt_d, ba_frames_d = _stage(dev, perm, seg, src, rig * ip, rig * jp + (ip == jp).long(),
                                                                   torch.unique(ii_ba))

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
    They run graphs whose update_op is droid_slam_b200.update.UpdateModule, whose tensors are on CUDA and which have edges; any other
    graph follows the strict policy (module docstring)."""
    unsupported = lambda graph, *args, **kwargs: _factor_graph_unsupported(graph)          # noqa: E731
    _replace(factor_graph_class, "update", _update, unsupported, strict)
    _replace(factor_graph_class, "update_lowmem", _update_lowmem, unsupported, strict)
    _record("install_factor_graph_hook", factor_graph_class, strict=strict)
    return factor_graph_class


# ---- PoseTrajectoryFiller ------------------------------------------------------------------------------------------------------------

_FILL_UPDATES = 6     # graph.update(N, N+M, motion_only=True) calls per batch (trajectory_filler.py:78-79)
_FNET_IMAGES = 16     # images per fnet call: the reference's batch


def _filler_unsupported(filler):
    """why fill_trajectory cannot run this PoseTrajectoryFiller natively (None: it can)"""
    why = _graph_unsupported("filler", filler, "update", ("fnet",), video=("poses", "disps", "intrinsics", "tstamp", "fmaps", "nets", "inps"))
    if why is None and filler.video.counter.value < 1:
        return "the video has no keyframe"
    return why


def _filler_frame_budget(be, ht, wd, device):
    """the most frames one fill_trajectory batch takes: a quarter of the free device memory over what one frame needs -- two edges, each
    with its volume pyramid (f16, four levels), its share of the update operator's workspace, its corr features, hidden state and outputs;
    and the frame's image (64 hw pixels x 3 channels) as uint8 on the device (fnet normalises it on load), its feature map (f16, 128
    channels) and its pose / intrinsics rows"""
    hw = ht * wd
    volume = 2 * sum(hw * (ht >> l) * (wd >> l) for l in range(4))
    per_edge = volume + _update_edge_bytes(be, ht, wd) + hw * (196 * 2 + 128 * 2 * 3 + 2 * 2 * 4 * 4 + 4 * 4)
    per_image = 64 * hw * 3 + hw * 128 * 2 + 4 * (7 + 4)
    return _quarter_free(device, 2 * per_edge + per_image)


def _fill_batch(be, filler, tstamps, images, intrinsics):
    """PoseTrajectoryFiller.__fill (trajectory_filler.py:42-84) for one batch of any size, with one host read -> (poses [M,7] on the
    device, the host copies of t0 and t1 [M] and of the edge list ii / jj in combined-frame indices).
    Frames [0, B) of the combined state are the video's buffer slots, frames [B, B+M) this batch; the video is only read."""
    video = filler.video
    dev = video.poses.device
    N, B, M = video.counter.value, video.poses.shape[0], len(tstamps)
    num, rig, ch, ht, wd = video.fmaps.shape
    tt = _stage(dev, torch.as_tensor(tstamps))
    images = _stage(dev, torch.stack(images, 0))
    intr = _stage(dev, torch.stack(intrinsics, 0)) / 8.0
    norm = _frame_norm(filler)
    cams, H, W = images.shape[1], images.shape[-2], images.shape[-1]
    fmap = torch.cat([_encode_frames(be, filler.fnet, images[a:a + _FNET_IMAGES].reshape(-1, 3, H, W), norm).view(-1, cams, ch, ht, wd)
                      for a in range(0, M, _FNET_IMAGES)])
    t0, t1, G = be.fill_interpolate(video.poses[:N].contiguous(), video.tstamp[:N].contiguous(), tt.float().contiguous())

    host = torch.stack([t0, t1]).cpu()                                   # the one host read: the edge list
    k = torch.arange(M)
    two = host[1] != host[0]                 # add_factors(t1, ...) drops the duplicates of the t0 edges (__filter_repeated_edges)
    ii = torch.cat([host[0], host[1][two]])
    jj = torch.cat([k, k[two]])
    ii = torch.where(ii < 0, ii + B, ii)     # t0 = -1: the reference's graph indexes slot -1 of the video's buffers, the last one
    E = ii.numel()
    ii_d, jj_d, jloc_d = _stage(dev, ii, jj + B, jj)

    with torch.autocast("cuda", enabled=False):
        poses = torch.cat([video.poses, G])
        intr_all = torch.cat([video.intrinsics, intr.float()])
        f1 = video.fmaps[:, 0]
        if f1.is_contiguous():
            vol_i = ii_d
        else:                                # stereo buffers: gather the edges' left images
            f1, vol_i = video.fmaps[ii_d, 0], torch.arange(E, device=dev)
        pyr, tiled = _volumes(be, f1, fmap[:, 0].contiguous(), vol_i, jloc_d)
        target = be.reproject(poses, video.disps, intr_all, ii_d, jj_d)[0]
        weight = torch.zeros_like(target)
        net, inp = video.nets[ii_d][None], video.inps[ii_d][None]
        ba_target = torch.empty(E, 2, ht, wd, device=dev)
        ba_weight = torch.empty_like(ba_target)
        damping = torch.empty(1, ht, wd, device=dev)                    # graph_writeback's shape argument; motion-only BA has no eta
        intr0 = video.intrinsics[0].contiguous()
        for _ in range(_FILL_UPDATES):
            coords, coords_t, motn = be.motion_features(poses, video.disps, intr_all, ii_d, jj_d, target)
            corr = _lookup(be, pyr, tiled, coords_t)
            net, delta, w = filler.update.forward_segments(net, inp, corr, motn[None], None, 0)
            be.graph_writeback(delta[0], w[0], coords, None, target, weight, ba_target, ba_weight, 0, None, None, damping, None, None, 0.0)
            be.pose_only_ba(poses, video.disps, intr0, ba_target, ba_weight, ii_d, jj_d, B, B + M, 2, 1e-4, 0.1, False)
    return poses[B:], (host[0], host[1], ii, jj + B)


def fill_trajectory(filler, image_stream):
    """PoseTrajectoryFiller.__call__ (reference trajectory_filler.py:86-110) on the native kernels -> poses [T,7] of every frame of the
    stream, `filler` being the reference's PoseTrajectoryFiller (or an object with its attributes: fnet, update, video, MEAN, STDV).

    Same steps per frame as the reference: pose interpolation between the bracketing keyframes (droid_backends.fill_interpolate), fnet,
    the edges from the keyframes t0 and t1 to the frame, their correlation volumes, initial targets from the reprojection, then six times
    the motion features, the corr lookup, the update operator (no GraphAgg: the filler graph neither upsamples nor uses eta) and two
    Gauss-Newton iterations of motion-only BA (droid_backends.pose_only_ba).  Every frame is independent of the others, so frames are
    batched by free device memory instead of by 16; one host read per batch.  Differences from the reference: the video is left as it
    was (the reference leaves the last batch in slots [N, N+16)), and a frame whose damped pose block is not positive definite keeps its
    pose in that iteration on its own (the reference zeroes the update of its whole 16-frame batch).  Raises when the filler cannot run
    natively (see install_trajectory_filler_hook)."""
    _require("PoseTrajectoryFiller.__call__", _filler_unsupported(filler))
    return _fill_trajectory(filler, image_stream)


def _fill_trajectory(filler, image_stream):
    be = install()
    video = filler.video
    budget = _filler_frame_budget(be, video.fmaps.shape[3], video.fmaps.shape[4], video.poses.device)
    out, batch = [], ([], [], [])
    with torch.no_grad():
        for tstamp, image, intrinsic in image_stream:
            for lst, x in zip(batch, (tstamp, image, intrinsic)):
                lst.append(x)
            if len(batch[0]) == budget:
                out.append(_fill_batch(be, filler, *batch)[0])
                batch = ([], [], [])
        if batch[0]:
            out.append(_fill_batch(be, filler, *batch)[0])
    return torch.cat(out) if out else video.poses.new_zeros(0, 7)


def install_trajectory_filler_hook(trajectory_filler_module, strict=True):
    """trajectory_filler_module = the imported reference module `trajectory_filler`.  Replaces `PoseTrajectoryFiller.__call__` by
    fill_trajectory; the result is an SE3 of that module's own lietorch, as the reference returns.  It runs fillers whose update operator
    is droid_slam_b200.update.UpdateModule, whose fnet is a BasicEncoder under install_encoder_hook and whose video tensors are on CUDA,
    with at least one keyframe; any other filler follows the strict policy (module docstring)."""
    _replace(trajectory_filler_module.PoseTrajectoryFiller, "__call__",
             lambda filler, image_stream: trajectory_filler_module.SE3(_fill_trajectory(filler, image_stream)),
             lambda filler, *args, **kwargs: _filler_unsupported(filler), strict)
    _record("install_trajectory_filler_hook", trajectory_filler_module, strict=strict)
    return trajectory_filler_module


# ---- MotionFilter ----------------------------------------------------------------------------------------------------------------------

def _motion_filter_unsupported(be, filt, image):
    """why track cannot run this MotionFilter on this frame natively (None: it can)"""
    why = _graph_unsupported("filter", filt, "update", ("fnet", "cnet"), video=("tstamp", "images", "poses", "disps", "disps_sens",
                                                                              "intrinsics", "fmaps", "nets", "inps"))
    if why is not None:
        return why
    if not (isinstance(image, torch.Tensor) and image.dim() == 4 and image.shape[1] == 3 and image.dtype == torch.uint8):
        return "the image must be a uint8 tensor [cameras,3,H,W]"
    H, W = image.shape[-2:]
    if H % 8 or W % 8:
        return "%dx%d images (H and W must be multiples of 8)" % (H, W)
    if H < 64 or W < 64 or not be.corr_volume_supported(128, H // 8, W // 8):
        return "no correlation volume kernel for %dx%d feature maps" % (H // 8, W // 8)
    return None


def _probe_grid(filt, ht, wd, dev):
    """the identity grid pops.coords_grid(ht, wd) as [1,2,ht,wd] (x, y) and the one-entry index of the probe's volume, cached per size"""
    key = (ht, wd, str(dev))
    cached = getattr(filt, "_b200_probe_grid", None)
    if cached is None or cached[0] != key:
        y, x = torch.meshgrid(torch.arange(ht, device=dev).float(), torch.arange(wd, device=dev).float(), indexing="ij")
        cached = (key, torch.stack([x, y])[None].contiguous(), torch.zeros(1, dtype=torch.long, device=dev))
        filt._b200_probe_grid = cached
    return cached[1], cached[2]


def _context(be, filt, frames, norm):
    """MotionFilter.__context_encoder (motion_filter.py:39-43) on camera 0 of the frames: net, inp [1,128,ht,wd] f16"""
    out = _encode_frames(be, filt.cnet, frames[:1], norm)
    net, inp = out[None].split([128, 128], dim=2)
    return net.tanh().squeeze(0), inp.relu().squeeze(0)


def track(filt, tstamp, image, depth=None, intrinsics=None):
    """MotionFilter.track (reference motion_filter.py:50-91) with the same signature and effects, `filt` being the reference's MotionFilter
    (or an object with its attributes: fnet, cnet, update, video, thresh, count, MEAN, STDV) -- the filter's net, inp, fmap and count and
    the video's buffers and counter, bit for bit as the reference method on the same operators.

    Per frame: the frame goes up through pinned staging without blocking; fnet takes the uint8 frames as stored (the BGR -> RGB flip and
    the normalisation happen in its first kernel, droid_backends.encoder_forward_frames); the motion probe builds the correlation volume
    of the last keyframe's and this frame's camera-0 features (corr_volume_pyramid) and looks it up on the identity grid
    (corr_lookup_pyramid), as CorrBlock under install_corr_volume_hook does; the update operator runs once without aggregation; the
    statistic is the reference's own `delta.norm(dim=-1).mean()`, and reading it is the one host read of the frame.  A keyframe (the
    statistic strictly above thresh, or the video's first frame) runs cnet on camera 0 and goes through `video.append`, so the video's lock
    and counter logic stay the video's.  Kept from the reference: the first frame writes net[0,0] / inp[0,0] (channel 0, broadcast over
    the video's 128 channels) and the identity pose and disparity 1.0; later keyframes write neither pose nor disparity; the depth
    (RGB-D) goes to the video as given, whose setter samples and inverts it; intrinsics are divided by 8.  Raises when the filter or the
    frame cannot run natively (see install_motion_filter_hook)."""
    _require("MotionFilter.track", _motion_filter_unsupported(install(), filt, image))
    _track(filt, tstamp, image, depth, intrinsics)


def _track(filt, tstamp, image, depth=None, intrinsics=None):
    be = install()
    video = filt.video
    dev = video.poses.device
    ht, wd = image.shape[-2] // 8, image.shape[-1] // 8
    norm = _frame_norm(filt)
    with torch.no_grad():
        frames = _stage(dev, image)
        gmap = _encode_frames(be, filt.fnet, frames, norm)                     # [cameras,128,ht,wd]
        if video.counter.value == 0:
            keyframe, pose, disp = True, video.poses.new_zeros(7), 1.0
            pose[6] = 1                                                         # lietorch.SE3.Identity(1).data
        else:
            coords_t, idx = _probe_grid(filt, ht, wd, dev)
            pyr, tiled = _volumes(be, filt.fmap[:1].contiguous(), gmap[:1].contiguous(), idx, idx)
            corr = _lookup(be, pyr, tiled, coords_t)
            _, delta, _ = filt.update.forward_segments(filt.net[None], filt.inp[None], corr, None, None, 0)
            with torch.autocast("cuda", enabled=True):
                stat = delta.norm(dim=-1).mean()
            keyframe, pose, disp = stat.item() > filt.thresh, None, None         # the one host read
        if not keyframe:
            filt.count += 1
            return
        with torch.autocast("cuda", enabled=True):
            net, inp = _context(be, filt, frames, norm)
        first = pose is not None
        if not first:
            filt.count = 0
        filt.net, filt.inp, filt.fmap = net, inp, gmap
        if depth is not None:
            depth = _stage(dev, depth)
        intr = _stage(dev, intrinsics) / 8.0
        # the stamp as a device scalar: the video's `tstamp[i] = stamp` then copies on the device instead of synchronising the host
        ts = _stage(dev, torch.as_tensor(tstamp, dtype=video.tstamp.dtype))
        video.append(ts, frames[0], pose, disp, depth, intr, gmap, net[0, 0] if first else net[0], inp[0, 0] if first else inp[0])


def install_motion_filter_hook(motion_filter_module, strict=True):
    """motion_filter_module = the imported reference module `motion_filter`.  Replaces `MotionFilter.track` (motion_filter.py:50-91) by
    track above.  It runs filters whose update operator is droid_slam_b200.update.UpdateModule, whose fnet and cnet are BasicEncoders
    under install_encoder_hook and whose video tensors are on CUDA, on uint8 frames [cameras,3,H,W] whose size the correlation kernels
    take; any other filter or frame follows the strict policy (module docstring)."""
    be = install()
    _replace(motion_filter_module.MotionFilter, "track", _track,
             lambda filt, tstamp, image, *args, **kwargs: _motion_filter_unsupported(be, filt, image), strict)
    _record("install_motion_filter_hook", motion_filter_module, strict=strict)
    return motion_filter_module


# ---- the hook registry and DroidAsync's backend process -----------------------------------------------------------------------------

_HOOKS = []        # every hook installed in this process, in order (see hook_registry)


def _resolve(module, qualname):
    """the module `module` (qualname None) or the object at `qualname` in it, importing the module"""
    obj = importlib.import_module(module)
    for part in (qualname.split(".") if qualname else ()):
        obj = getattr(obj, part)
    return obj


def _record(installer, target, **kwargs):
    """enter the hook `installer(target, **kwargs)` in the registry.  target is transferable when it is a module or a class that another
    interpreter finds by name: the module sys.modules holds under its name, or the class at its qualified name in such a module"""
    module, qualname = getattr(target, "__module__", None), getattr(target, "__qualname__", None)
    if isinstance(target, types.ModuleType):
        module, qualname = target.__name__, None
    transferable = isinstance(target, (types.ModuleType, type)) and module in sys.modules and "<locals>" not in (qualname or "")
    if transferable:
        try:
            transferable = _resolve(module, qualname) is target
        except AttributeError:
            transferable = False
    entry = {"installer": installer, "module": module, "qualname": qualname, "kwargs": kwargs, "transferable": transferable,
             "target": "%s.%s" % (module, qualname) if qualname else (module if transferable else repr(target))}
    if transferable:                     # installing again on the same target replaces the entry
        _HOOKS[:] = [e for e in _HOOKS if not (e["transferable"] and (e["installer"], e["module"], e["qualname"]) == (installer, module, qualname))]
    _HOOKS.append(entry)


def hook_registry():
    """a copy of the registry: per installed hook, in installation order, a dict of installer (the install_* function's name), module
    (the importable name of the reference module patched, or of the module defining the patched class), qualname (the class's qualified
    name; None when the module itself was passed), kwargs (strict, fused_lookup), transferable (False for a target another interpreter
    cannot find by name, e.g. a SimpleNamespace) and target (a readable name).  Plain data: it pickles."""
    return copy.deepcopy(_HOOKS)


def _installer(name):
    """the function a registry entry's installer names: an install_* hook of this module, or the package's install_dependencies (which
    takes no target)"""
    if name == "install_dependencies":
        from . import install_dependencies
        return lambda target, **kwargs: install_dependencies()
    return globals()[name]


def reinstall_hooks(hooks):
    """install every transferable hook of `hooks` (as hook_registry gives them) in this interpreter, by module name, in order"""
    install()
    for e in hooks:
        if e["transferable"]:
            _installer(e["installer"])(_resolve(e["module"], e["qualname"]), **e["kwargs"])


def install_update_module_hook(droid_net_module):
    """droid_net_module = the imported reference module `droid_net`.  Sets its global `UpdateModule` (droid_net.py:111-143) to
    droid_slam_b200.update.UpdateModule, so `DroidNet()` -- and both reference `load_network` functions, which build it -- construct the
    native update operator.  Same parameter names: a DROID checkpoint loads unchanged (the callers already slice the heads to 2 rows)."""
    from .update import UpdateModule
    droid_net_module.UpdateModule = UpdateModule
    _record("install_update_module_hook", droid_net_module)
    return droid_net_module


# the hooks the native backend loop runs on: DroidAsyncBackend -> FactorGraph.add_proximity_factors / update_lowmem(use_inactive=True)
# on AltCorrBlock and DepthVideo.reproject / upsample, with the network's update operator
_BACKEND_HOOKS = ("install_update_module_hook", "install_factor_graph_hook", "install_alt_corr_hook", "install_proximity_hook",
                  "install_depth_video_hook")
_HANDOVER_BUFFERS = ("poses", "disps", "disps_sens", "images", "tstamp", "intrinsics", "fmaps", "nets", "inps")


def _async_unsupported(hooks):
    """why a spawned backend process cannot run natively with these hooks (None: it can)"""
    lost = [e["installer"] + " on " + e["target"] for e in hooks if not e["transferable"]]
    if lost:
        return "hooks on objects a spawned process cannot import by name: " + ", ".join(lost)
    missing = [h for h in _BACKEND_HOOKS if not any(e["installer"] == h for e in hooks)]
    if missing:
        return "the native backend needs " + ", ".join(missing)
    return None


def handover_round(video1, video2, t0, t1, diagnostics=False):
    """the hand-over of one backend round (reference droid_async.py:54-119) on droid_backends.fragment_handover: under video1's lock,
    the slices [t0,t1) of video1's buffers go to video2, the fragment alignment and the re-anchoring of poses / disps run on video2's
    device, and the lock is released after one synchronisation of video2's device's current stream -- the round's one host sync.
    t0 == 0 or t0 >= 10 (what backend_process produces).  Returns the diagnostics [9] f64 (s, dG, align_scale) when asked, else None."""
    be = install()
    with video1.get_lock():
        out = be.fragment_handover([getattr(video1, k) for k in _HANDOVER_BUFFERS], [getattr(video2, k) for k in _HANDOVER_BUFFERS],
                                   int(t0), int(t1), bool(video2.stereo), diagnostics)
        torch.cuda.current_stream(video2.poses.device).synchronize()
    return out[0] if diagnostics else None


_BACKEND_ITERS_SHARED, _BACKEND_ITERS_OWN_DEVICE = 8, 12   # global-BA iterations per round: backend on the frontend's GPU / on its own
_BACKEND_START_FRAMES = 32          # the frontend's keyframe count above which rounds start before the end of the stream
_BACKEND_FRONTIER_GAP = 5           # keyframes left to the frontend's local window in a round before the last
_BACKEND_OVERLAP = 2                # keyframes of the previous round handed over again (t0 = counter2 - 2)
_BACKEND_PAUSE_S = 10               # seconds between rounds while the stream lasts


def _backend_loop(mod, args, front, back, device="cuda"):
    """The decisions of the reference's backend_process (droid_async.py:37-130), with the hand-over on handover_round.

    device "cuda" shares the frontend's GPU (8 iterations per round); any other device string is selected for this process and gets 12
    (:40-50).  Rounds run while the frontend holds more than 32 keyframes or the stream has ended (back.ready, :55); a round hands over
    keyframes [max(back.counter - 2, 0), t1) with t1 = the frontend's counter in the final round and 5 fewer before it (:57-71), sets
    back.counter = t1 and calls the backend with normalize=False (:121-122).  The final round ends the loop; otherwise, unless the stream
    ended meanwhile, the loop waits 10 s (:124-128).  load_network and DroidAsyncBackend are looked up in `mod`, as the reference's
    module globals are."""
    torch.set_num_threads(8)
    own_device = device != "cuda"
    if own_device:
        torch.cuda.set_device(device)
    iters = _BACKEND_ITERS_OWN_DEVICE if own_device else _BACKEND_ITERS_SHARED
    with torch.no_grad():
        ba = mod.DroidAsyncBackend(mod.load_network(args.weights, device=device), back, args)
        while True:
            if not (front.counter.value > _BACKEND_START_FRAMES or back.ready.value):
                continue                                           # the reference polls without pausing here too
            final = bool(back.ready.value)                         # read again, as the reference does
            first = max(back.counter.value - _BACKEND_OVERLAP, 0)
            end = front.counter.value - (0 if final else _BACKEND_FRONTIER_GAP)
            handover_round(front, back, first, end)
            back.counter.value = end
            ba(iters, normalize=False)
            if final:
                return
            if back.ready.value <= 0:
                time.sleep(_BACKEND_PAUSE_S)


def _unpickle_backend(module, strict, reference, hooks, native):
    """a BackendProcess as a spawned interpreter unpickles it.  The Process object pickles its target before its arguments, so this runs
    before DepthVideo is unpickled -- which imports the reference's depth_video and, with it, `lietorch`: a recorded install_dependencies
    therefore registers the packages here, not in prepare()"""
    if any(e["installer"] == "install_dependencies" and e["transferable"] for e in hooks or ()):
        from . import install_dependencies
        install_dependencies()
    return BackendProcess(module, strict, reference, hooks, native)


class BackendProcess:
    """The `backend_process` install_async_hook puts into the reference's droid_async module; DroidAsync starts it as a Process target.

    Pickled (which is how `spawn` hands it to the new interpreter) it carries the hook registry of that moment, checked first: a hook on
    an object that cannot be imported by name, or a missing hook of the native backend (_BACKEND_HOOKS), raises under strict=True --
    in the parent, as DroidAsync starts the process -- and makes the child run the reference's own backend_process under strict=False.
    In the child, unpickling runs a recorded install_dependencies first (_unpickle_backend); __call__ runs droid_slam_b200.install(),
    re-installs every recorded hook by module name, then the native loop.  Called
    without pickling (in the installing process, or a forked child, where the hooks are in place) it checks the same and runs the loop."""

    def __init__(self, module, strict=True, reference=None, hooks=None, native=None):
        self.module, self.strict, self.reference, self.hooks, self.native = module, strict, reference, hooks, native

    def __reduce__(self):
        if self.native is not None:                          # already a snapshot
            return _unpickle_backend, (self.module, self.strict, None, self.hooks, self.native)
        why = _async_unsupported(_HOOKS)
        if why is not None and self.strict:
            _require("droid_async.backend_process", why)
        return _unpickle_backend, (self.module, self.strict, None, hook_registry(), why is None)

    def prepare(self):
        """install the native extension and the carried hooks in this interpreter -> the droid_async module"""
        reinstall_hooks(self.hooks)
        return importlib.import_module(self.module)

    def __call__(self, args, depth_video1, depth_video2, device="cuda"):
        if self.native is None:                              # not pickled: the hooks of this process apply
            why = _async_unsupported(_HOOKS)
            if why is not None and not self.strict:
                return self.reference(args, depth_video1, depth_video2, device)
            _require("droid_async.backend_process", why)
            return _backend_loop(importlib.import_module(self.module), args, depth_video1, depth_video2, device)
        if not self.native:                                  # a fresh interpreter: its droid_async holds the reference's function
            return importlib.import_module(self.module).backend_process(args, depth_video1, depth_video2, device)
        return _backend_loop(self.prepare(), args, depth_video1, depth_video2, device)


def install_async_hook(droid_async_module, strict=True):
    """droid_async_module = the imported reference module `droid_async`.  Replaces its global `backend_process` (droid_async.py:37-130,
    the target of DroidAsync's backend Process) by a BackendProcess: in the spawned process it re-installs every hook recorded in this
    process (hook_registry) and runs the reference's loop with the hand-over on handover_round.  Under strict=True, starting DroidAsync
    raises when a recorded hook cannot be re-installed by name or a hook the native backend needs is missing (_BACKEND_HOOKS);
    strict=False then keeps the reference's backend_process."""
    ref = droid_async_module.backend_process
    if isinstance(ref, BackendProcess):
        ref = ref.reference
    droid_async_module.backend_process = BackendProcess(droid_async_module.__name__, strict, ref)
    return droid_async_module


# ---- the differentiable dense BA layer under DroidNet ----------------------------------------------------------------------------------

BA_LAYER_MAX_POSES = 20       # pose unknowns (N - fixedp) the layer factors in one launch (include/droid_b200.h DBA_BA_LAYER_MAX_POSES)
_BA_EP, _BA_LM = 0.1, 1e-4    # schur_solve's damping (geom/chol.py:46)


class _BALayer(torch.autograd.Function):
    """geom/ba.py BA on droid_backends.ba_layer_forward / ba_layer_backward.  The forward keeps the fp64 factor, dx, dz and the flags;
    the backward recomputes the per-pixel terms.  intrinsics, ii and jj get no gradient."""

    @staticmethod
    def forward(ctx, target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp):
        be = install()
        out = be.ba_layer_forward(target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp, _BA_EP, _BA_LM, False)
        ctx.fixedp = fixedp
        ctx.save_for_backward(target, weight, eta, poses, disps, intrinsics, ii, jj, *out[2:])
        return out[0], out[1]

    @staticmethod
    def backward(ctx, grad_poses, grad_disps):
        target, weight, eta, poses, disps, intrinsics, ii, jj, factor, dx, dz, flags = ctx.saved_tensors
        gp = torch.zeros_like(poses) if grad_poses is None else grad_poses.contiguous()
        gd = torch.zeros_like(disps) if grad_disps is None else grad_disps.contiguous()
        g = install().ba_layer_backward(gp, gd, target, weight, eta, poses, disps, intrinsics, ii, jj, ctx.fixedp, _BA_EP, _BA_LM,
                                        factor, dx, dz, flags)
        return g[0], g[1], g[2], g[3], g[4], None, None, None, None


def _ba_layer_unsupported(target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp=1, rig=1):
    """why the native layer cannot run this BA call, or None"""
    if type(poses).__name__ != "SE3" or not hasattr(poses, "data") or poses.data.shape[-1:] != (7,):
        return "poses must be SE3 (got %s)" % type(poses).__name__
    if rig != 1:
        return "rig = %r (only rig = 1)" % (rig,)
    N = disps.shape[1] if torch.is_tensor(disps) and disps.dim() == 4 else 0
    if not 0 <= fixedp < N:
        return "fixedp = %r outside [0, N) = [0, %d)" % (fixedp, N)
    named = (("target", target), ("weight", weight), ("eta", eta), ("poses", poses.data), ("disps", disps), ("intrinsics", intrinsics))
    for name, t in named:
        if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32):
            return "%s must be a CUDA float32 tensor" % name
    if intrinsics.requires_grad:
        return "intrinsics requires grad (the layer gives it none)"
    if N - fixedp > BA_LAYER_MAX_POSES:
        return "%d pose unknowns, more than the %d one launch factors" % (N - fixedp, BA_LAYER_MAX_POSES)
    return None


def ba_layer(target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp=1, rig=1):
    """BA(target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp=1, rig=1) of geom/ba.py:31-106 -> (poses', disps'), poses' of
    the caller's SE3 class, differentiable in target, weight, eta, poses (every frame) and disps.  One autograd Function over the
    native forward and backward; under no_grad (or with no input requiring grad) nothing is kept.  No host synchronisation."""
    _require("BA", _ba_layer_unsupported(target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp, rig))
    dev = disps.device
    ii = ii.to(device=dev, dtype=torch.long).contiguous()
    jj = jj.to(device=dev, dtype=torch.long).contiguous()
    args = (target.contiguous(), weight.contiguous(), eta.contiguous(), poses.data.contiguous(), disps.contiguous(), intrinsics.contiguous())
    if torch.is_grad_enabled() and any(t.requires_grad for t in args):
        p, d = _BALayer.apply(*args, ii, jj, int(fixedp))
    else:
        p, d = install().ba_layer_forward(*args, ii, jj, int(fixedp), _BA_EP, _BA_LM, False)[:2]
    return type(poses)(p), d


def install_ba_layer_hook(droid_net_module, strict=True):
    """droid_net_module = the imported reference module `droid_net`.  Sets its global `BA` (droid_net.py:13, called twice per update
    iteration in DroidNet.forward) to the native layer (`ba_layer`), forward and backward.  A call the layer cannot run (poses not SE3,
    tensors not CUDA float32, rig != 1, fixedp outside [0, N), intrinsics requiring grad, more than BA_LAYER_MAX_POSES pose unknowns)
    raises under strict=True and runs the reference's BA under strict=False."""
    _replace(droid_net_module, "BA", ba_layer, _ba_layer_unsupported, strict)
    _record("install_ba_layer_hook", droid_net_module, strict=strict)
    return droid_net_module


# ---- the differentiable CorrBlock under DroidNet -----------------------------------------------------------------------------------

class _CorrGrad:
    """one training block's gradient pyramid [E,ht*wd,Q] during a backward pass (None outside one).  The backward contexts hold only
    this, not the block's volumes, which no backward reads."""

    def __init__(self):
        self.gpyr = None


class _CorrBuild(torch.autograd.Function):
    """fmap1, fmap2 [E,128,ht,wd] f32 -> a token every lookup takes as an input.  Autograd runs this backward after every lookup that
    reaches the loss has added its gradient into the block's gradient pyramid: the adjoint runs once, and the pyramid is released so
    that the next backward pass starts from zero."""

    @staticmethod
    def forward(ctx, fmap1, fmap2, state):
        ctx.state = state                      # a _CorrGrad
        ctx.save_for_backward(fmap1, fmap2)
        return fmap1.new_zeros(0)

    @staticmethod
    def backward(ctx, _):
        fmap1, fmap2 = ctx.saved_tensors
        state = ctx.state
        if state.gpyr is None:                 # no lookup reached the loss
            return torch.zeros_like(fmap1), torch.zeros_like(fmap2), None
        g1, g2 = install().corr_adjoint(fmap1, fmap2, state.gpyr)
        state.gpyr = None
        return g1, g2, None


class _CorrLookup(torch.autograd.Function):
    """one CorrBlock.__call__: coords [E,2,ht,wd] -> [E,196,ht,wd]; its backward adds into the block's gradient pyramid (zeroed by the
    first lookup of a backward pass) and gives the token a zero gradient, coords none"""

    @staticmethod
    def forward(ctx, token, coords, pyramid, state):
        ctx.state = state                      # a _CorrGrad
        ctx.save_for_backward(coords)
        return install().corr_lookup_pyramid(pyramid, coords)

    @staticmethod
    def backward(ctx, grad):
        coords, = ctx.saved_tensors
        state = ctx.state
        if state.gpyr is None:
            E, _, ht, wd = coords.shape
            q = sum((ht >> l) * (wd >> l) for l in range(4))
            state.gpyr = torch.zeros(E, ht * wd, q, dtype=torch.float32, device=coords.device)
        install().corr_grad_accumulate(coords, grad.contiguous(), state.gpyr)
        return coords.new_zeros(0), None, None, None


def _corr_training_unsupported(fmap1, fmap2, num_levels=4, radius=3):
    """why the native training CorrBlock cannot run these arguments (None: it can)"""
    why = _corr_fmaps_unsupported(fmap1, fmap2, num_levels)
    if why is not None:
        return why
    if fmap1.dtype != torch.float32 or fmap2.dtype != torch.float32:
        return "dtype %s / %s (float32 has a kernel)" % (fmap1.dtype, fmap2.dtype)
    if radius != 3:
        return "radius %d (3 has a kernel)" % radius
    batch, num = fmap1.shape[:2]
    if batch * num > 65535:
        return "%d edges (at most 65535)" % (batch * num)
    return None


class CorrBlock:
    """CorrBlock(fmap1, fmap2, num_levels=4, radius=3) of modules/corr.py:6-71 for fp32 [B,N,128,ht,wd] CUDA feature maps, differentiable
    in both maps: the volume and its pooled levels (`droid_backends.corr_volume_pyramid_f32`), each call's 4-level lookup
    (`corr_lookup_pyramid`, bit-identical to the reference's corr_index_forward + cat on these volumes) and one backward per pass
    (`corr_grad_accumulate` per call into one gradient pyramid, `corr_adjoint` once).  coords get no gradient, as in the reference.
    Under no_grad, or with maps that do not require grad, nothing is kept for backward.  No host synchronisation."""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        _require("CorrBlock", _corr_training_unsupported(fmap1, fmap2, num_levels, radius))
        be = install()
        self.num_levels, self.radius = num_levels, radius
        batch, num, dim, ht, wd = fmap1.shape
        f1 = fmap1.reshape(batch * num, dim, ht, wd).contiguous()
        f2 = fmap2.reshape(batch * num, dim, ht, wd).contiguous()
        self.corr_pyramid = be.corr_volume_pyramid_f32(f1.detach(), f2.detach())
        self._grad = _CorrGrad()
        self._token = None
        if torch.is_grad_enabled() and (f1.requires_grad or f2.requires_grad):
            self._token = _CorrBuild.apply(f1, f2, self._grad)

    def __call__(self, coords):
        batch, num, ht, wd, _ = coords.shape
        c = coords.detach().permute(0, 1, 4, 2, 3).contiguous().view(batch * num, 2, ht, wd).float()
        if self._token is not None and torch.is_grad_enabled():
            out = _CorrLookup.apply(self._token, c, self.corr_pyramid, self._grad)
        else:
            out = install().corr_lookup_pyramid(self.corr_pyramid, c)
        return out.view(batch, num, -1, ht, wd)


def install_corr_training_hook(droid_net_module, strict=True):
    """droid_net_module = the imported reference module `droid_net`.  Sets its global `CorrBlock` (droid_net.py:8, built once per
    DroidNet.forward and looked up once per update iteration) to the native training block (`CorrBlock` above), forward and backward.
    A block it cannot build (not fp32 CUDA [B,N,128,ht,wd] maps with ht, wd >= 8, num_levels != 4, radius != 3; f16 / autocast training
    among them) raises under strict=True and builds the reference's CorrBlock under strict=False.  modules.corr.CorrBlock, which the
    frontend, the factor graph and the motion filter use, is not touched."""
    _replace(droid_net_module, "CorrBlock", CorrBlock, _corr_training_unsupported, strict)
    _record("install_corr_training_hook", droid_net_module, strict=strict)
    return droid_net_module


# ---- training's tail under the reference's losses / droid_net: the flow loss and upsample_disp ----------------------------------------

def _se3_data(P):
    """P's [..., 7] data when P is an SE3, else None"""
    data = getattr(P, "data", None) if type(P).__name__ == "SE3" else None
    return data if torch.is_tensor(data) and data.shape[-1:] == (7,) else None


def _f32_cuda(t):
    return torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32


def _flow_loss_unsupported(Ps, disps, poses_est, disps_est, intrinsics, graph=None, gamma=0.9):
    """why the native flow loss cannot run this call, or None"""
    if _se3_data(Ps) is None:
        return "Ps must be an SE3 [B,N,7] (got %s)" % type(Ps).__name__
    if len(poses_est) == 0 or len(poses_est) != len(disps_est):
        return "%d pose and %d disparity iterates (the same number, at least one, has a kernel)" % (len(poses_est), len(disps_est))
    for k, P in enumerate(poses_est):
        if _se3_data(P) is None:
            return "poses_est[%d] must be an SE3 [B,N,7] (got %s)" % (k, type(P).__name__)
    named = [("Ps", Ps.data), ("disps", disps), ("intrinsics", intrinsics)]
    named += [("poses_est[%d]" % k, P.data) for k, P in enumerate(poses_est)] + [("disps_est[%d]" % k, d) for k, d in enumerate(disps_est)]
    for name, t in named:
        if not _f32_cuda(t):
            return "%s must be a CUDA float32 tensor" % name
    if disps.dim() != 4:
        return "disps must be [B,N,ht,wd] (got shape %s)" % (tuple(disps.shape),)
    B, N, ht, wd = disps.shape
    for name, t in named:
        want = (B, N, 7) if name.startswith(("Ps", "poses_est")) else (B, N, 4) if name == "intrinsics" else (B, N, ht, wd)
        if tuple(t.shape) != want:
            return "%s has shape %s, not %s" % (name, tuple(t.shape), want)
    if N < 2:
        return "N = %d (the chain graph needs 2 frames)" % N
    if B * ht * wd == 0:
        return "an empty batch or image"
    for name, t in (("Ps", Ps.data), ("disps", disps), ("intrinsics", intrinsics)):
        if t.requires_grad:
            return "%s requires grad (the native loss gives it none)" % name
    return None


class _FlowLoss(torch.autograd.Function):
    """geom/losses.py flow_loss on droid_backends.flow_loss_forward / flow_loss_backward over the 2n iterate tensors (poses' data,
    then disparities).  Nothing but the inputs is kept: the backward recomputes every per-pixel term."""

    @staticmethod
    def forward(ctx, Ps, disps, intrinsics, gamma, *est):
        n = len(est) // 2
        loss, metrics = install().flow_loss_forward(Ps, disps, list(est[:n]), list(est[n:]), intrinsics, gamma)
        ctx.gamma = gamma
        ctx.save_for_backward(Ps, disps, intrinsics, *est)
        ctx.mark_non_differentiable(metrics)
        return loss, metrics

    @staticmethod
    def backward(ctx, grad_loss, _):
        Ps, disps, intrinsics, *est = ctx.saved_tensors
        n = len(est) // 2
        g = install().flow_loss_backward(grad_loss.reshape(()).float().contiguous(), Ps, disps, est[:n], est[n:], intrinsics, ctx.gamma)
        return (None, None, None, None, *g)


def flow_loss(Ps, disps, poses_est, disps_est, intrinsics, graph=None, gamma=0.9):
    """flow_loss(Ps, disps, poses_est, disps_est, intrinsics, graph, gamma=0.9) of geom/losses.py:89-118 -> (loss, metrics): every
    iterate in one pass over the full-resolution pixels of the chain graph (graph is ignored, as the reference ignores it), nothing
    materialised per pixel; differentiable in every poses_est[i] (lietorch's convention) and disps_est[i].  metrics is the reference's
    dict of Python floats ('f_error', '1px': NaN when no pixel is valid, as the mean of an empty tensor) from one host read."""
    _require("flow_loss", _flow_loss_unsupported(Ps, disps, poses_est, disps_est, intrinsics, graph, gamma))
    args = (Ps.data.contiguous(), disps.contiguous(), intrinsics.contiguous())
    est = [P.data.contiguous() for P in poses_est] + [d.contiguous() for d in disps_est]
    if torch.is_grad_enabled() and any(t.requires_grad for t in est):
        loss, metrics = _FlowLoss.apply(*args, float(gamma), *est)
    else:
        n = len(poses_est)
        loss, metrics = install().flow_loss_forward(*args[:2], est[:n], est[n:], args[2], float(gamma))
    s, count, below = metrics.tolist()
    nan = float("nan")
    return loss, {"f_error": s / count if count else nan, "1px": below / count if count else nan}


def install_flow_loss_hook(losses_module, strict=True):
    """losses_module = the imported reference module `geom.losses`.  Sets its global `flow_loss` (losses.py:89, which train.py calls
    through the module) to the native loss (`flow_loss`), forward and backward.  A call it cannot run (Ps or a poses_est[i] not an SE3
    [B,N,7], a tensor not CUDA float32, shapes that disagree, N < 2, no iterates, Ps / disps / intrinsics requiring grad) raises under
    strict=True and runs the reference's flow_loss under strict=False.  projective_transform itself is not touched."""
    _replace(losses_module, "flow_loss", flow_loss, _flow_loss_unsupported, strict)
    _record("install_flow_loss_hook", losses_module, strict=strict)
    return losses_module


def _upsample_disp_unsupported(disp, mask):
    """why the native upsample_disp cannot run this call, or None"""
    if not (_f32_cuda(disp) and disp.dim() == 4):
        return "disp must be a CUDA float32 [B,N,ht,wd] tensor"
    B, N, ht, wd = disp.shape
    if not (_f32_cuda(mask) and tuple(mask.shape) == (B, N, 576, ht, wd)):
        return "mask must be a CUDA float32 [B,N,576,ht,wd] = %s tensor (got %s %s)" % (
            (B, N, 576, ht, wd), getattr(mask, "dtype", type(mask).__name__), tuple(getattr(mask, "shape", ())))
    return None


class _UpsampleDisp(torch.autograd.Function):
    """droid_net.py upsample_disp on droid_backends.cvx_upsample and cvx_upsample_backward; disp [n,ht,wd], mask [n,576,ht,wd]"""

    @staticmethod
    def forward(ctx, disp, mask):
        ctx.save_for_backward(disp, mask)
        return install().cvx_upsample(disp, mask)

    @staticmethod
    def backward(ctx, grad):
        disp, mask = ctx.saved_tensors
        return tuple(install().cvx_upsample_backward(disp, mask, grad.contiguous()))


def upsample_disp(disp, mask):
    """upsample_disp(disp, mask) of droid_net.py:37-42 for fp32 CUDA inputs: disp [B,N,ht,wd], mask [B,N,576,ht,wd] -> [B,N,8ht,8wd],
    the forward droid_backends.cvx_upsample's, differentiable in both (the softmax recomputed from the mask, nothing else kept)"""
    _require("upsample_disp", _upsample_disp_unsupported(disp, mask))
    B, N, ht, wd = disp.shape
    d = disp.reshape(B * N, ht, wd).contiguous()
    m = mask.reshape(B * N, 576, ht, wd).contiguous()
    if torch.is_grad_enabled() and (d.requires_grad or m.requires_grad):
        out = _UpsampleDisp.apply(d, m)
    else:
        out = install().cvx_upsample(d, m)
    return out.view(B, N, 8 * ht, 8 * wd)


def install_upsample_disp_hook(droid_net_module, strict=True):
    """droid_net_module = the imported reference module `droid_net`.  Sets its global `upsample_disp` (droid_net.py:37, called once per
    update iteration by DroidNet.forward) to the native one (`upsample_disp`), forward and backward.  A call with a disp that is not a
    CUDA float32 [B,N,ht,wd] or a mask that is not a CUDA float32 [B,N,576,ht,wd] raises under strict=True and runs the reference's
    upsample_disp under strict=False."""
    _replace(droid_net_module, "upsample_disp", upsample_disp, _upsample_disp_unsupported, strict)
    _record("install_upsample_disp_hook", droid_net_module, strict=strict)
    return droid_net_module


# ---- the update operator's ConvGRU under modules.gru -------------------------------------------------------------------------------

# ConvGRU(128, 128+128+64) as UpdateModule builds it: the parameters' names, in the order droid_backends.conv_gru_* take them
CONV_GRU_PARAMS = ("convz.weight", "convz.bias", "convr.weight", "convr.bias", "convq.weight", "convq.bias", "w.weight", "w.bias",
                   "convz_glo.weight", "convz_glo.bias", "convr_glo.weight", "convr_glo.bias", "convq_glo.weight", "convq_glo.bias")


def _conv_gru_params(module):
    return [module.get_parameter(name) for name in CONV_GRU_PARAMS]


def _conv_gru_unsupported(module, net, *inputs):
    """why the native ConvGRU cannot run this call (None: it can)"""
    convs = [getattr(module, name.split(".")[0], None) for name in CONV_GRU_PARAMS[::2]]
    want = [(128, 448, 3)] * 3 + [(128, 128, 1)] * 4
    got = [(c.out_channels, c.in_channels, c.kernel_size[0]) if isinstance(c, torch.nn.Conv2d) else None for c in convs]
    if got != want or any(c.bias is None for c in convs):
        return "the module is not ConvGRU(128, 320): (out, in, kernel) of its convolutions are %s, not %s" % (got, want)
    tensors = [("net", net)] + [("inputs[%d]" % k, t) for k, t in enumerate(inputs)]
    if not all(torch.is_tensor(t) for _, t in tensors):
        return "net and the inputs must be tensors"
    channels = tuple(t.shape[1] if t.dim() == 4 else None for _, t in tensors)
    if channels != (128, 128, 128, 64):
        return "net and inputs must be 4-d with 128 / (128, 128, 64) channels, got %s" % (channels,)
    shapes = {(t.shape[0],) + tuple(t.shape[2:]) for _, t in tensors}
    if len(shapes) > 1:
        return "net and the inputs disagree in (b, h, w): %s" % sorted(shapes)
    b, h, w = shapes.pop()
    if b * h * w == 0:
        return "an empty batch or image"
    if b > 65535 or b * 448 * h * w >= 2 ** 31:
        return "%d edges of %dx%d (at most 65535 edges and b * 448 * h * w < 2^31)" % (b, h, w)
    named = tensors + list(zip(CONV_GRU_PARAMS, _conv_gru_params(module)))
    for name, t in named:
        if not _f32_cuda(t):
            return "%s must be a CUDA float32 tensor (got %s on %s)" % (name, t.dtype, t.device)
    devs = {t.device for _, t in named}
    if len(devs) > 1:
        return "the tensors and parameters are on %d devices (%s), not one" % (len(devs), ", ".join(sorted(map(str, devs))))
    if torch.is_autocast_enabled("cuda"):
        return "CUDA autocast is enabled (the reference would run float16 convolutions)"
    return None


class _ConvGRU(torch.autograd.Function):
    """modules/gru.py ConvGRU.forward on droid_backends.conv_gru_forward / conv_gru_backward.  The parameters are inputs, so autograd
    accumulates their .grad.  The forward keeps z, r, q (384 channels) and glo beyond the inputs and parameters."""

    @staticmethod
    def forward(ctx, net, inp, corr, flow, *params):
        out, zr, q, glo = install().conv_gru_forward(net, inp, corr, flow, list(params))
        ctx.save_for_backward(net, inp, corr, flow, zr, q, glo, *params)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad):
        net, inp, corr, flow, zr, q, glo, *params = ctx.saved_tensors
        return tuple(install().conv_gru_backward(grad.contiguous(), net, inp, corr, flow, params, zr, q, glo))


def conv_gru(module, net, *inputs):
    """ConvGRU.forward(net, *inputs) of modules/gru.py:19-32 for `module` = ConvGRU(128, 128+128+64) and fp32 CUDA tensors net
    [b,128,h,w], inputs (inp, corr, flow) [b,128|128|64,h,w] -> the new net [b,128,h,w], differentiable in net, the inputs and the
    module's 14 parameters (3xTF32 on the tensor cores, fixed-order sums: two runs give the same bits).  Non-contiguous tensors are
    copied.  Under no_grad, or with nothing requiring grad, nothing is kept.  No host synchronisation."""
    _require("ConvGRU.forward", _conv_gru_unsupported(module, net, *inputs))
    args = [t.contiguous() for t in (net,) + tuple(inputs)]
    params = _conv_gru_params(module)
    if torch.is_grad_enabled() and any(t.requires_grad for t in args + params):
        return _ConvGRU.apply(*args, *params)
    return install().conv_gru_forward(*args, [p.detach() for p in params])[0]


def install_conv_gru_hook(gru_module, strict=True):
    """gru_module = the imported reference module `modules.gru`.  Replaces `ConvGRU.forward` in place on the class (UpdateModule runs it
    once per update iteration, droid_net.py:127) by `conv_gru`, forward and backward.  A call it cannot run (not ConvGRU(128, 320), a
    tensor or parameter not CUDA float32 on one device, CUDA autocast enabled, other channel counts, mismatched b / h / w) raises under
    strict=True and runs the reference's forward under strict=False.  The inference operator's install_update_module_hook replaces the
    whole UpdateModule, so a network built under it never calls ConvGRU.forward."""
    _replace(gru_module.ConvGRU, "forward", conv_gru, _conv_gru_unsupported, strict)
    _record("install_conv_gru_hook", gru_module, strict=strict)
    return gru_module
