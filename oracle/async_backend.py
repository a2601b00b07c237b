"""DroidAsync's frontend -> backend hand-over, restated on the lietorch stand-in (oracle/shims/lietorch) -- TEST INFRASTRUCTURE ONLY.

  * align_pose_fragments: the Sim(3) fragment alignment of reference droid_slam/align.py:3-24 (`align_pose_fragements`), with the same
    group operations in the same order, in the dtype of its inputs.  tests/golden/make_async_golden.py pins it bit
    for bit against the unmodified file.
  * handover: one round of backend_process's hand-over, reference droid_slam/droid_async.py:54-119, on dicts of the two videos'
    buffers (poses, disps, disps_sens, images, tstamp, intrinsics, fmaps, nets, inps); returns the back buffers after the round and what
    the alignment gave.
  * reanchor: the re-anchoring of droid_async.py:87, :94-96 (dG composed with the frontend's poses whose translations were scaled by s
    in fp32), composed in fp64 and rounded once (what dba_fragment_handover computes).
"""
import torch

from .shims.lietorch import SE3

BUFFERS = ("poses", "disps", "disps_sens", "images", "tstamp", "intrinsics", "fmaps", "nets", "inps")


def _pair_translations(G):
    """the translation of G[j]^-1 G[i] for every pair (i, j) of the group batch G [n], as [n*n, 3]"""
    return (G[None, :].inv() * G[:, None]).data[..., :3].reshape(-1, 3)


def align_pose_fragments(src, dst):
    """align.py:3-24 -> (g SE3 [1], scale 0-dim tensor): the scale that fits src's pairwise translations to dst's in least squares, and
    the pose g that maps the scaled src fragment onto dst (its first pair, then 3 refinements by the mean of the log residuals).  Same
    group operations in the same order as the reference, in the dtype of the inputs."""
    a, b = SE3(src.clone()), SE3(dst.clone())
    ta, tb = _pair_translations(a), _pair_translations(b)
    scale = (ta * tb).sum() / (ta * ta).sum()
    a.data[..., :3] *= scale             # g is fitted to the scaled fragment whether or not the caller keeps the scale
    g = (b * a.inv())[[0]]
    for _ in range(3):
        residual = (b * (g * a).inv()).log()
        g = SE3.exp(residual.mean(dim=0, keepdim=True)) * g
    return g, scale


def handover(front, back, t0, t1, stereo, align_dtype=None):
    """One round's hand-over, droid_async.py:54-119 -> (back buffers after the round as new tensors, s, dG data [1,7], align_scale).

    front / back: dicts of the BUFFERS.  The scale is kept only without stereo and without any nonzero sensor depth anywhere in the
    frontend's buffer; with t0 > 0 the frontend's fragment [t0-10, t0-1) is aligned to the backend's (in align_dtype, default the poses'
    dtype); t0 == 0 is the identity with scale 1.  Frames [t0,t1) of the frontend, translations scaled, are composed with dG in the poses'
    dtype, their inverse depths divided by the scale, and the other buffers copied.  s is the float 1.0 where the scale is not kept."""
    after = {k: v.clone() for k, v in back.items()}
    keep_scale = not stereo and not bool(torch.any(front["disps_sens"]))
    poses, dtype = front["poses"].clone(), front["poses"].dtype
    if t0 == 0:
        dG, s = SE3.IdentityLike(SE3(back["poses"][[0]])), 1.0
    else:
        work = align_dtype or dtype
        dG, s = align_pose_fragments(poses[t0 - 10:t0 - 1].to(work), back["poses"][t0 - 10:t0 - 1].to(work))
        s = s if keep_scale else 1.0
    applied = s.to(dtype) if isinstance(s, torch.Tensor) else s
    poses[..., :3] *= applied
    after["poses"][t0:t1] = (SE3(dG.data.to(dtype)) * SE3(poses[t0:t1])).data
    after["disps"][t0:t1] = front["disps"][t0:t1] / applied
    for k in BUFFERS[2:]:
        after[k][t0:t1] = front[k][t0:t1]
    return after, s, dG.data, keep_scale


def reanchor(poses, s, dG):
    """dG * SE3(poses with translations * float32(s)) in fp64 from the fp32 poses, rounded once to fp32.  poses [n,7] f32, s a float,
    dG [7]"""
    p = poses.float().clone()
    p[:, :3] *= torch.tensor(s, dtype=torch.float32)
    g = SE3(torch.as_tensor(dG, dtype=torch.float64).reshape(1, 7)) * SE3(p.double())
    return g.data.float()
