"""time corr_volume_pyramid (wgmma) against the reference formula on the GPU (cuBLAS fp16 matmul + 3x avg_pool2d)"""
import os, sys, json, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import droid_slam_b200
be = droid_slam_b200.install()
dev = "cuda"
E = int(sys.argv[1]) if len(sys.argv) > 1 else 128
N, C, ht, wd = 72, 128, 48, 64
g = torch.Generator().manual_seed(0)
fmaps = torch.randn(N, C, ht, wd, generator=g).half().to(dev)
ii = torch.randint(0, N, (E,), generator=g).to(dev); jj = torch.randint(0, N, (E,), generator=g).to(dev)
def timeit(fn, n=10, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
def ref():
    f1 = fmaps[ii].reshape(E, C, ht * wd) / 4.0; f2 = fmaps[jj].reshape(E, C, ht * wd) / 4.0
    corr = torch.matmul(f1.transpose(1, 2), f2).reshape(E * ht * wd, 1, ht, wd)
    pyr = []
    for l in range(4):
        pyr.append(corr.view(E, ht, wd, ht >> l, wd >> l))
        corr = torch.nn.functional.avg_pool2d(corr, 2, stride=2)
    return pyr
t_ours = timeit(lambda: be.corr_volume_pyramid(fmaps, fmaps, ii, jj))
t_ref = timeit(ref)
HW = ht * wd
bytes_written = E * HW * HW * 2 * (1 + 1 / 4 + 1 / 16 + 1 / 64)
flops = 2.0 * E * HW * HW * C
print(json.dumps({"E": E, "ours_ms": t_ours, "ref_ms": t_ref, "speedup": t_ref / t_ours, "ours_write_GBps": bytes_written / t_ours / 1e6,
                  "ours_TFLOPs": flops / t_ours / 1e9, "ref_write_GBps_algorithmic": bytes_written / t_ref / 1e6}))
