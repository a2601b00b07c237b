"""Restatement of the data flow of FactorGraph.update and FactorGraph.update_lowmem (reference droid_slam/factor_graph.py:214-330)
-- TEST INFRASTRUCTURE ONLY.

Every operator is pluggable: the graph's own objects are called as the reference calls them -- `video.reproject(ii, jj)`,
`graph.corr(coords)` (update), `alt_corr_block(fmaps)(coords, ii, jj)` (update_lowmem), `graph.update_op(net, inp, corr, motn, ii, jj)`,
`video.ba(...)`, `video.upsample(ix, upmask)` -- so the same restatement runs on CPU stand-ins (pinned against the unmodified reference
methods by tests/golden/make_factor_graph_golden.py) and on the native kernels (the yardstick of the update / update_lowmem hooks).
Autocast regions of the reference are not restated: on CPU tensors and on the native operators they change nothing.

Reference behaviours kept on purpose:
  * t0 = max(1, ii.min() + 1) when not given (update);
  * update uses the inactive edges with ii_inac >= t0 - 3 and jj_inac >= t0 - 3, update_lowmem all of them; inactive edges come
    first in BA's inputs;
  * damping[unique(ii)] = eta, then BA gets .2 * damping[unique(ii of BA's edges)] + EP;
  * age += 1 per update and per update_lowmem step, video.dirty[:t] = True per update_lowmem step;
  * BA: update (t0, t1, lm=1e-4, ep=0.1, motion_only), update_lowmem (1, t, lm=1e-5, ep=1e-2);
  * AltCorrBlock indices rig * ii, rig * jj + (ii == jj);
  * update_lowmem chunks start at range(ii.min(), jj.max() + 1, 8): an edge whose source frame lies beyond the last chunk is not
    passed to the update operator (its net, target and weight keep their values) but still enters BA.
"""
import torch

__all__ = ["CHUNK_FRAMES", "motion_features", "update", "update_lowmem", "lowmem_chunk_starts"]

CHUNK_FRAMES = 8


def motion_features(coords1, coords0, target):
    """[1,E,ht,wd,2] x3 -> motn [1,E,4,ht,wd]: (coords1 - grid, target - coords1) clamped to +-64"""
    flow = torch.cat([coords1 - coords0, target - coords1], dim=-1)
    return flow.permute(0, 1, 4, 2, 3).clamp(-64.0, 64.0)


def lowmem_chunk_starts(ii, jj):
    """first source frame of every update_lowmem chunk (each spans CHUNK_FRAMES source frames)"""
    return list(range(int(ii.min()), int(jj.max()) + 1, CHUNK_FRAMES))


def _channels_first(x, ht, wd):
    return x.view(-1, ht, wd, 2).permute(0, 3, 1, 2).contiguous()


def _bundle_adjust(graph, inactive, EP, t0, t1, itrs, lm, ep, motion_only):
    """BA over the inactive edges selected by `inactive` (bool mask or None) followed by the active ones"""
    ht, wd = graph.coords0.shape[:2]
    if inactive is None:
        ii, jj, target, weight = graph.ii, graph.jj, graph.target, graph.weight
    else:
        ii = torch.cat([graph.ii_inac[inactive], graph.ii])
        jj = torch.cat([graph.jj_inac[inactive], graph.jj])
        target = torch.cat([graph.target_inac[:, inactive], graph.target], dim=1)
        weight = torch.cat([graph.weight_inac[:, inactive], graph.weight], dim=1)
    damping = 0.2 * graph.damping[torch.unique(ii)].contiguous() + EP
    graph.video.ba(_channels_first(target, ht, wd), _channels_first(weight, ht, wd), damping, ii, jj, t0, t1,
                   itrs=itrs, lm=lm, ep=ep, motion_only=motion_only)


def update(graph, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
    video = graph.video
    coords1, _ = video.reproject(graph.ii, graph.jj)
    motn = motion_features(coords1, graph.coords0, graph.target)
    corr = graph.corr(coords1)
    graph.net, delta, weight, eta, upmask = graph.update_op(graph.net, graph.inp, corr, motn, graph.ii, graph.jj)
    if t0 is None:
        t0 = max(1, int(graph.ii.min()) + 1)
    graph.target = coords1 + delta.float()
    graph.weight = weight.float()
    graph.damping[torch.unique(graph.ii)] = eta
    inactive = None
    if use_inactive:
        inactive = (graph.ii_inac >= t0 - 3) & (graph.jj_inac >= t0 - 3)
    _bundle_adjust(graph, inactive, EP, t0, t1, itrs, 1e-4, 0.1, motion_only)
    if graph.upsample:
        video.upsample(torch.unique(graph.ii), upmask)
    graph.age += 1


def update_lowmem(graph, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, steps=8, alt_corr_block=None):
    """alt_corr_block: the AltCorrBlock class (the reference takes it from its module's imports)"""
    video = graph.video
    t = video.counter.value
    num, rig, ch, ht, wd = video.fmaps.shape
    corr_op = alt_corr_block(video.fmaps.view(1, num * rig, ch, ht, wd))
    for _ in range(steps):
        coords1, _ = video.reproject(graph.ii, graph.jj)
        motn = motion_features(coords1, graph.coords0, graph.target)
        for first in lowmem_chunk_starts(graph.ii, graph.jj):
            sel = (graph.ii >= first) & (graph.ii < first + CHUNK_FRAMES)
            if not bool(sel.any()):
                continue
            src, dst = graph.ii[sel], graph.jj[sel]
            corr = corr_op(coords1[:, sel], rig * src, rig * dst + (src == dst).long())
            net, delta, weight, eta, upmask = graph.update_op(graph.net[:, sel], video.inps[None, src], corr, motn[:, sel], src, dst)
            if graph.upsample:
                video.upsample(torch.unique(src), upmask)
            graph.net[:, sel] = net
            graph.target[:, sel] = coords1[:, sel] + delta.float()
            graph.weight[:, sel] = weight.float()
            graph.damping[torch.unique(src)] = eta
        graph.age += 1
        everything = torch.ones_like(graph.ii_inac, dtype=torch.bool) if use_inactive else None
        _bundle_adjust(graph, everything, EP, 1, t, itrs, 1e-5, 1e-2, False)
        video.dirty[:t] = True
