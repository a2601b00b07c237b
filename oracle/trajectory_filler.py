"""Restatement of PoseTrajectoryFiller.__fill / __call__ (reference droid_slam/trajectory_filler.py:42-110) -- TEST INFRASTRUCTURE ONLY.

Every operator is pluggable, as in oracle/factor_graph.py: the SE3 class (lietorch, or the stand-in under oracle/shims), the filler's
own fnet / update operator, and the factor graph made by `make_graph(video, update_op)` with the reference's `add_factors` / `update`
methods.  The video is the caller's object with DepthVideo's buffers, `counter` and `__setitem__`.

Reference behaviours kept on purpose:
  * t0 = #{k < N : ts[k] <= t} - 1 without assuming ts is sorted; t1 = t0 + 1 if t0 < N - 1 else t0;
  * t0 = -1 (a frame stamped before keyframe 0): P[t0] and ts[t0] are keyframe N - 1 (Python indexing), the graph's edge -1 -> frame
    indexes slot -1 of the video's buffers;
  * edges: add_factors(t0, frames) then add_factors(t1, frames), which drops the duplicates when t0 == t1;
  * 6 x graph.update(N, N + M, motion_only=True); batches of 16 frames; the batch is written into video slots [N, N + M) and counter is
    restored afterwards (the slots keep the last batch).
"""
import torch

__all__ = ["BATCH", "interpolate", "fill_batch", "fill", "FillerGraph"]

BATCH = 16


class FillerGraph:
    """FactorGraph as __fill uses it (factor_graph.py:20-53, 95-150): a fresh graph, `add_factors` with `__filter_repeated_edges` against
    the active edges, volume correlation (`corr_block(fmap1, fmap2)` and its `cat`), no factor limit; `update(t0, t1, motion_only=...)`
    calls `update_fn(graph, ...)` (oracle.factor_graph.update, or a hook)."""

    def __init__(self, video, update_op, corr_block, update_fn, device="cpu"):
        self.video, self.update_op, self.device, self.upsample = video, update_op, device, False
        self._corr_block, self._update_fn = corr_block, update_fn
        ht, wd = video.disps.shape[1:]
        y, x = torch.meshgrid(torch.arange(ht, device=device).float(), torch.arange(wd, device=device).float(), indexing="ij")
        self.coords0 = torch.stack([x, y], dim=-1)
        z = torch.zeros(0, dtype=torch.long, device=device)
        self.ii, self.jj, self.age, self.ii_inac, self.jj_inac = z, z, z, z, z
        self.corr = self.net = self.inp = None
        self.damping = 1e-6 * torch.ones_like(video.disps)
        self.target = torch.zeros(1, 0, ht, wd, 2, device=device)
        self.weight = torch.zeros(1, 0, ht, wd, 2, device=device)
        self.target_inac = torch.zeros(1, 0, ht, wd, 2, device=device)
        self.weight_inac = torch.zeros(1, 0, ht, wd, 2, device=device)

    def add_factors(self, ii, jj, remove=False):
        if len(self.ii) > 0:
            mask = ((ii[:, None] == self.ii) & (jj[:, None] == self.jj)).any(dim=-1)
            ii, jj = ii[~mask], jj[~mask]
        if ii.shape[0] == 0:
            return
        v = self.video
        net = v.nets[ii].to(self.device).unsqueeze(0)
        c = (ii == jj).long()
        corr = self._corr_block(v.fmaps[ii, 0].to(self.device).unsqueeze(0), v.fmaps[jj, c].to(self.device).unsqueeze(0))
        self.corr = corr if self.corr is None else self.corr.cat(corr)
        inp = v.inps[ii].to(self.device).unsqueeze(0)
        self.inp = inp if self.inp is None else torch.cat([self.inp, inp], 1)
        target, _ = v.reproject(ii, jj)
        weight = torch.zeros_like(target)
        self.ii = torch.cat([self.ii, ii], 0)
        self.jj = torch.cat([self.jj, jj], 0)
        self.age = torch.cat([self.age, torch.zeros_like(ii)], 0)
        self.net = net if self.net is None else torch.cat([self.net, net], 1)
        self.target = torch.cat([self.target, target], 1)
        self.weight = torch.cat([self.weight, weight], 1)

    def update(self, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
        self._update_fn(self, t0, t1, itrs=itrs, use_inactive=use_inactive, EP=EP, motion_only=motion_only)


def interpolate(poses, ts, tstamps, SE3):
    """trajectory_filler.py:51-65: poses [N,7] and ts [N] of the keyframes, tstamps (a list) -> (t0, t1 int64 [M], G [M,7])"""
    N = poses.shape[0]
    tt = torch.as_tensor(tstamps, device=poses.device)
    Ps = SE3(poses)
    t0 = torch.as_tensor([ts[ts <= t].shape[0] - 1 for t in tstamps])
    t1 = torch.where(t0 < N - 1, t0 + 1, t0)
    dt = ts[t1] - ts[t0] + 1e-3
    dP = Ps[t1] * Ps[t0].inv()
    v = dP.log() / dt.unsqueeze(-1)
    w = v * (tt - ts[t0]).unsqueeze(-1)
    Gs = SE3.exp(w) * Ps[t0]
    return t0, t1, Gs.data


def fill_batch(filler, tstamps, images, intrinsics, make_graph, SE3):
    """__fill: -> (poses [M,7], graph ii, graph jj)"""
    video = filler.video
    dev = video.poses.device
    tt = torch.as_tensor(tstamps, device=dev)
    images = torch.stack(images, 0).to(dev)
    intrinsics = torch.stack(intrinsics, 0)
    inputs = images[:, :, [2, 1, 0]] / 255.0
    N = video.counter.value
    M = len(tstamps)
    t0, t1, G = interpolate(video.poses[:N], video.tstamp[:N], tstamps, SE3)
    inputs = inputs.sub_(filler.MEAN).div_(filler.STDV)
    with torch.autocast("cuda", enabled=dev.type == "cuda"):
        fmap = filler.fnet(inputs)
    video.counter.value += M
    video[N:N + M] = (tt, images[:, 0], G, 1, None, intrinsics.to(dev) / 8.0, fmap)
    graph = make_graph(video, filler.update)
    graph.add_factors(t0.to(dev), torch.arange(N, N + M, device=dev))
    graph.add_factors(t1.to(dev), torch.arange(N, N + M, device=dev))
    for _ in range(6):
        graph.update(N, N + M, motion_only=True)
    out = video.poses[N:N + M].clone()
    video.counter.value -= M
    return out, graph.ii.clone(), graph.jj.clone()


def fill(filler, image_stream, make_graph, SE3, batch=BATCH):
    """__call__: -> (poses [T,7], per batch (ii, jj))"""
    poses, edges, cur = [], [], ([], [], [])
    for item in image_stream:
        for lst, x in zip(cur, item):
            lst.append(x)
        if len(cur[0]) == batch:
            p, ii, jj = fill_batch(filler, *cur, make_graph, SE3)
            poses.append(p); edges.append((ii, jj))
            cur = ([], [], [])
    if cur[0]:
        p, ii, jj = fill_batch(filler, *cur, make_graph, SE3)
        poses.append(p); edges.append((ii, jj))
    return torch.cat(poses), edges
