"""Host side of the native feature / context encoders: `BasicEncoder.forward` (reference droid_slam/modules/extractor.py:118-198) for
DroidNet's fnet = BasicEncoder(128, 'instance') and cnet = BasicEncoder(256, 'none') on the kernels of `csrc/encoder.cu` (C ABI
`dba_encoder_forward`, include/droid_b200.h).  The reference module keeps its own parameters; `modules.install_encoder_hook` routes its
forward here.

`pack_encoder_weights` only re-arranges the reference's parameters into the kernels' layout, f16 [taps][N][Kpad] (K contiguous, zero
padded to a multiple of 64) plus f32 biases, in the order of `dba_encoder_weights`:

  0      conv1 7x7/2 3->32 as one 1x1 GEMM over the image im2col rows: [1][32][192], K = (dy*7 + dx)*3 + c
  1..4   layer1.{0,1}.{conv1,conv2}: [9][32][64] (tap = dy*3 + dx; K 32..63 zero, the kernels read 32-channel rows)
  5      layer2.0: conv1 (3x3/2) and downsample.0 (1x1/2) as one 1x1 GEMM over the gathered 3x3/2 taps: [1][128][320] with
         K = (dy*3 + dx)*32 + c; rows 0..63 = conv1, rows 64..127 = the downsample in the centre-tap rows K 128..159
  6..8   layer2.0.conv2, layer2.1.{conv1,conv2}: [9][64][64]
  9      layer3.0: conv1 | downsample.0 like 5: [1][256][576], K = (dy*3 + dx)*64 + c, downsample in K 256..319
  10..12 layer3.0.conv2, layer3.1.{conv1,conv2}: [9][128][128]
  13     conv2 1x1 128->output_dim: [1][output_dim][128]
"""
import torch

__all__ = ["pack_encoder_weights", "ENCODER_CONVS"]

# state_dict prefixes of the 14 GEMMs; layer2.0 / layer3.0 conv1 also carry their downsample
ENCODER_CONVS = ("conv1", "layer1.0.conv1", "layer1.0.conv2", "layer1.1.conv1", "layer1.1.conv2", "layer2.0.conv1", "layer2.0.conv2",
                 "layer2.1.conv1", "layer2.1.conv2", "layer3.0.conv1", "layer3.0.conv2", "layer3.1.conv1", "layer3.1.conv2", "conv2")


def _taps(w):
    """[Co,Ci,k,k] -> [k*k (dy*k + dx), Co, Kpad], K = input channel, zero padded to a multiple of 64"""
    co, ci, k, _ = w.shape
    t = w.permute(2, 3, 0, 1).reshape(k * k, co, ci)
    kpad = -(-ci // 64) * 64
    return torch.cat([t, t.new_zeros(k * k, co, kpad - ci)], 2)


def _gathered(w, wd):
    """3x3/2 conv1 [P,C,3,3] and 1x1/2 downsample [P,C,1,1] -> [1][2P][Kpad]: K = (dy*3 + dx)*C + c, the downsample on the centre tap"""
    p, c = w.shape[0], w.shape[1]
    kpad = -(-9 * c // 64) * 64
    out = w.new_zeros(2 * p, kpad)
    out[:p, :9 * c] = w.permute(0, 2, 3, 1).reshape(p, 9 * c)
    out[p:, 4 * c:5 * c] = wd[:, :, 0, 0]
    return out[None]


def pack_encoder_weights(sd, norm_fn, output_dim, device=None):
    """state_dict of a reference BasicEncoder (norm_fn 'instance' or 'none', output_dim 128 or 256) -> list of 28 tensors: the 14 packed
    f16 weights, then the 14 f32 biases (layouts: module docstring).  Pure re-arrangement; the norm layers have no parameters."""
    if norm_fn not in ("instance", "none"):
        raise ValueError("the native encoder has kernels for norm_fn 'instance' and 'none', not %r" % (norm_fn,))
    if output_dim not in (128, 256) or tuple(sd["conv2.weight"].shape[:2]) != (output_dim, 128):
        raise ValueError("conv2 must be 128 -> output_dim with output_dim 128 or 256")
    f = {k: v.detach().float().cpu() for k, v in sd.items()}
    ws, bs = [], []
    for name in ENCODER_CONVS:
        w, b = f[name + ".weight"], f[name + ".bias"]
        if name == "conv1":                                           # [32,3,7,7] -> K = (dy*7 + dx)*3 + c
            ws.append(torch.cat([w.permute(0, 2, 3, 1).reshape(32, 147), w.new_zeros(32, 45)], 1)[None])
        elif name in ("layer2.0.conv1", "layer3.0.conv1"):
            blk = name[:-len(".conv1")]
            ws.append(_gathered(w, f[blk + ".downsample.0.weight"]))
            b = torch.cat([b, f[blk + ".downsample.0.bias"]])
        else:
            ws.append(_taps(w))
        bs.append(b)
    out = [t.to(torch.float16).contiguous() for t in ws] + [t.to(torch.float32).contiguous() for t in bs]
    return [t.to(device) for t in out] if device is not None else out
