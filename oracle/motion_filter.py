"""Restatement of MotionFilter.track (reference droid_slam/motion_filter.py:50-91) -- TEST INFRASTRUCTURE ONLY.

Every operator is pluggable, as in oracle/trajectory_filler.py: the filter's own fnet / cnet / update operator, the correlation block
`corr_block(fmap1, fmap2)` (called on the coordinate grid, as modules/corr.py's CorrBlock is) and the video, the caller's object with
DepthVideo's buffers, `counter` and `append`.  The filter is any object with MotionFilter's attributes (fnet, cnet, update, video,
thresh, count, device, MEAN, STDV).

Reference behaviours kept on purpose:
  * the frame is flipped BGR -> RGB and normalised in fp32 by ATen: x / 255.0, .sub_(MEAN), .div_(STDV);
  * the video's first frame is always a keyframe and writes the identity pose, disparity 1.0 and net[0,0] / inp[0,0] (channel 0 of the
    context features, which the video's setter broadcasts over its 128 channels); the filter keeps the full maps and count is untouched;
  * later frames: the motion probe is one update-operator call on the correlation of the last keyframe's and this frame's camera-0
    features at the identity grid; a keyframe when delta.norm(dim=-1).mean() > thresh (strict), which resets count, writes neither pose
    nor disparity and net[0] / inp[0]; otherwise count += 1;
  * stereo: fnet runs on every camera, the probe and cnet on camera 0; depth goes to the video as given (its setter samples
    [3::8, 3::8] and inverts); intrinsics / 8.0.
"""
import torch

__all__ = ["track", "coords_grid", "IDENTITY"]

IDENTITY = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)     # lietorch.SE3.Identity(1,).data.squeeze()


def coords_grid(ht, wd, device):
    """geom/projective_ops.py coords_grid: [ht,wd,2], (x, y) per pixel"""
    y, x = torch.meshgrid(torch.arange(ht, device=device).float(), torch.arange(wd, device=device).float(), indexing="ij")
    return torch.stack([x, y], dim=-1)


def _context(filt, inputs):
    net, inp = filt.cnet(inputs).split([128, 128], dim=2)
    return net.tanh().squeeze(0), inp.relu().squeeze(0)


def track(filt, tstamp, image, depth=None, intrinsics=None, corr_block=None):
    """MotionFilter.track -> the motion statistic of the frame (a float; None for the video's first frame), with the reference's effects
    on the filter and the video.  The whole call runs under CUDA autocast, as the reference's decorator puts it, when the filter's
    device is a CUDA device."""
    dev = torch.device(filt.device)
    with torch.no_grad(), torch.autocast("cuda", enabled=dev.type == "cuda"):
        ht, wd = image.shape[-2] // 8, image.shape[-1] // 8
        image = image.to(dev)
        inputs = image[None, :, [2, 1, 0]] / 255.0
        inputs = inputs.sub_(filt.MEAN).div_(filt.STDV)
        gmap = filt.fnet(inputs).squeeze(0)
        video = filt.video
        if video.counter.value == 0:
            net, inp = _context(filt, inputs[:, [0]])
            filt.net, filt.inp, filt.fmap = net, inp, gmap
            video.append(tstamp, image[0], torch.tensor(IDENTITY), 1.0, depth, intrinsics / 8.0, gmap, net[0, 0], inp[0, 0])
            return None
        coords0 = coords_grid(ht, wd, dev)[None, None]
        corr = corr_block(filt.fmap[None, [0]], gmap[None, [0]])(coords0)
        _, delta, _ = filt.update(filt.net[None], filt.inp[None], corr)
        stat = delta.norm(dim=-1).mean().item()
        if stat > filt.thresh:
            filt.count = 0
            net, inp = _context(filt, inputs[:, [0]])
            filt.net, filt.inp, filt.fmap = net, inp, gmap
            video.append(tstamp, image[0], None, None, depth, intrinsics / 8.0, gmap, net[0], inp[0])
        else:
            filt.count += 1
        return stat
