"""Two calls of the tensor-core update operator at E edges (env UPD_E, default 256), 48x64, for a profiler to wrap: the first call is
the warm-up, the second the profiled one."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from droid_slam_b200 import synth
from droid_slam_b200.update import UpdateModule

DEV = "cuda:0"
E, ht, wd = int(os.environ.get("UPD_E", 256)), 48, 64
mod = UpdateModule().to(DEV); mod.load_state_dict(synth.make_update_weights(0))
g = torch.Generator(device=DEV).manual_seed(0)
net = torch.tanh(torch.randn(1, E, 128, ht, wd, device=DEV, generator=g)).half()
inp = torch.relu(torch.randn(1, E, 128, ht, wd, device=DEV, generator=g)).half()
corr = torch.randn(1, E, 196, ht, wd, device=DEV, generator=g).half()
flow = 4 * torch.randn(1, E, 4, ht, wd, device=DEV, generator=g)
ii = torch.arange(E, device=DEV) // 8
with torch.no_grad():
    for _ in range(int(os.environ.get("UPD_CALLS", 2))):
        out = mod(net, inp, corr, flow, ii)
torch.cuda.synchronize()
print("ok", float(out[0].float().abs().mean()))
