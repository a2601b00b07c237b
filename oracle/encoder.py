"""fp32 restatement of DroidNet's feature / context encoder, BasicEncoder (reference droid_slam/modules/extractor.py:118-198), for
norm_fn 'instance' (fnet) and 'none' (cnet), dropout 0, multidim False.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

`encoder_forward` follows the structure with F.conv2d / F.instance_norm; `BasicEncoder` is a stand-in with the reference's parameter
names and its `norm_fn` / `multidim` / `dropout` attributes, for tests of the hook where the reference tree is not available.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

__all__ = ["encoder_forward", "BasicEncoder"]


def _norm(x, norm_fn):
    # InstanceNorm2d(planes): affine=False, track_running_stats=False -> per-image statistics, biased variance, eps 1e-5
    # (extractor.py:28-32, 130-131); 'none' is an empty nn.Sequential (extractor.py:34-38, 133-134)
    return F.instance_norm(x, eps=1e-5) if norm_fn == "instance" else x


def _block(sd, pre, x, norm_fn, stride):
    """ResidualBlock.forward (extractor.py:47-55); the downsample is conv 1x1/stride + norm3 (:43-45)"""
    y = F.relu(_norm(F.conv2d(x, sd[pre + "conv1.weight"], sd[pre + "conv1.bias"], stride=stride, padding=1), norm_fn))
    y = F.relu(_norm(F.conv2d(y, sd[pre + "conv2.weight"], sd[pre + "conv2.bias"], padding=1), norm_fn))
    if stride != 1:
        x = _norm(F.conv2d(x, sd[pre + "downsample.0.weight"], sd[pre + "downsample.0.bias"], stride=stride), norm_fn)
    return F.relu(x + y)


def encoder_forward(sd, x, norm_fn):
    """BasicEncoder.forward (extractor.py:183-198): x [b,n,3,H,W] -> [b,n,output_dim,H/8,W/8], computed in x's dtype"""
    b, n, c, h, w = x.shape
    x = x.reshape(b * n, c, h, w)
    x = F.relu(_norm(F.conv2d(x, sd["conv1.weight"], sd["conv1.bias"], stride=2, padding=3), norm_fn))     # :187-189
    for layer in (1, 2, 3):                                                                                 # :191-193, _make_layer :175-181
        x = _block(sd, "layer%d.0." % layer, x, norm_fn, 1 if layer == 1 else 2)
        x = _block(sd, "layer%d.1." % layer, x, norm_fn, 1)
    x = F.conv2d(x, sd["conv2.weight"], sd["conv2.bias"])                                                  # :195
    return x.view(b, n, x.shape[1], x.shape[2], x.shape[3])


class _Block(nn.Module):
    def __init__(self, cin, p, norm_fn, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, p, 3, padding=1, stride=stride)
        self.conv2 = nn.Conv2d(p, p, 3, padding=1)
        self.downsample = nn.Sequential(nn.Conv2d(cin, p, 1, stride=stride), nn.Identity()) if stride != 1 else None


class BasicEncoder(nn.Module):
    """stand-in with the reference's constructor, parameter names and attributes; forward = encoder_forward on its own state_dict"""

    def __init__(self, output_dim=128, norm_fn="batch", dropout=0.0, multidim=False):
        super().__init__()
        self.norm_fn, self.multidim = norm_fn, multidim
        self.conv1 = nn.Conv2d(3, 32, 7, stride=2, padding=3)
        self.layer1 = nn.Sequential(_Block(32, 32, norm_fn, 1), _Block(32, 32, norm_fn, 1))
        self.layer2 = nn.Sequential(_Block(32, 64, norm_fn, 2), _Block(64, 64, norm_fn, 1))
        self.layer3 = nn.Sequential(_Block(64, 128, norm_fn, 2), _Block(128, 128, norm_fn, 1))
        self.conv2 = nn.Conv2d(128, output_dim, 1)
        self.dropout = nn.Dropout2d(p=dropout) if dropout > 0 else None

    def forward(self, x):
        return encoder_forward(self.state_dict(), x, self.norm_fn)
