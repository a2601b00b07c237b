"""The encoder kernels launch by launch through the C ABI (`dba_encoder_forward_prefix`), each checked by `check_stage` of
tests/test_encoder_stages_cpu.py (the references and bounds are derived there) on the workspace snapshots around it.

Per case and encoder: the workspace, a margin after it and the output start as NaN bytes; for k = 1 .. n_launches the first k launches
run and the workspace is snapshotted, stage k is checked on snapshot k - 1 -> k, every region stage k does not own (and its own regions
past the extent of its output) must be bit-identical between the two, the margin and the output's guards must stay untouched, and the
whole `dba_encoder_forward` must give the bits of the last prefix.  Non-finite inputs are checked end to end against which outputs of
the fp64 oracle are NaN.

Measured on one NVIDIA H100 80GB HBM3 at a 700 W power limit (name and limit read in the same run; this file and
tests/test_encoder_gpu.py together: 43 tests in 18 s).  Per case and encoder: the worst convolution kappa / sqrt(K) (the bound is 0.5)
and the smallest fraction of its outputs equal to the correctly rounded fp64 value; the activation pass's worst kappa (the bound is 4)
and fraction; the worst share of the slot, merge and whole-image statistics tolerances that was used (the bound is 1):
  384x512                fnet  0.199  0.9940   1.43  1.0000   0.32  0.08  0.12
  384x512                cnet  0.183  0.9970
  352x552                fnet  0.185  0.9940   1.66  1.0000   0.33  0.06  0.12
  352x552                cnet  0.179  0.9970
  384x512_shift40        fnet  0.194  0.9940   1.66  1.0000   0.53  0.03  0.11
  384x512_shift40        cnet  0.209  0.9980
  240x320_f16            fnet  0.208  0.9950   1.34  1.0000   0.28  0.09  0.12
  240x320_f16            cnet  0.173  0.9970
  8x8_n16                fnet  0.049  0.9980   0.42  1.0000   0.30  0.12  0.14
  8x8_n16                cnet  0.050  0.9990
  8x520_n2               fnet  0.137  0.9980   1.37  1.0000   0.27  0.06  0.08
  8x520_n2               cnet  0.144  0.9980
  24x72_n2_const1        fnet  0.090  0.9950   0.70  1.0000   0.32  0.09  0.12
  24x72_n2_const1        cnet  0.085  0.9980
  40x128_n2              fnet  0.143  0.9950   1.27  1.0000   0.28  0.08  0.13
  40x128_n2              cnet  0.126  0.9980
  64x96_n2_bias          fnet  0.142  0.9960   0.64  1.0000   0.22  0.10  0.14
  64x96_n2_bias          cnet  0.139  0.9980
  64x96_n16_f16_shift40  fnet  0.199  0.9950   1.43  1.0000   0.44  0.09  0.12
  64x96_n16_f16_shift40  cnet  0.155  0.9980
  128x256_n2             fnet  0.173  0.9940   1.53  1.0000   0.28  0.09  0.13
  128x256_n2             cnet  0.234  0.9970
Over all cases by K: 147: 0.157, 288: 0.234, 576: 0.199, 1152: 0.172, conv2 (K = 128): 0.209 sqrt(K)."""
import ctypes
import json
import os

import pytest
import torch

import oracle.encoder as oenc
from droid_slam_b200 import c_api, synth
from droid_slam_b200.encoder import pack_encoder_weights
from test_encoder_stages_cpu import CASES, CASE_IDS, ENCODERS, bits, case_images, case_weights, check_stage, layout, stage_table
from util import card, stream

pytestmark = pytest.mark.gpu
dev = "cuda"
GUARD = 64                      # fp16 elements of NaN before and after the output
MARGIN = 4096                   # NaN bytes after the workspace


class Run:
    """one encoder call set up in guarded NaN-filled buffers: `prefix(k)` runs the first k launches, `forward()` all of them"""

    def __init__(self, L, name, sd, images):
        self.L = L
        self.norm, self.od = ENCODERS[name]
        n, _, H, W = images.shape
        self.lay = layout(L, n, H, W, self.norm)
        self.images = images.to(dev).contiguous()
        self.pk = pack_encoder_weights(sd, "instance" if self.norm else "none", self.od, dev)
        self.wt = c_api.EncoderWeights()
        for k in range(14):
            self.wt.w[k], self.wt.b[k] = self.pk[k].data_ptr(), self.pk[14 + k].data_ptr()
        total = self.lay["total"]
        self.buf = torch.full((total + MARGIN,), 255, dtype=torch.uint8, device=dev)
        assert self.buf.data_ptr() % 256 == 0
        self.ws = self.buf[:total]
        self.shape = (n, self.od, H // 8, W // 8)
        self.out = self.new_out()

    def new_out(self):
        n = self.shape[0] * self.shape[1] * self.shape[2] * self.shape[3]
        return torch.full((n + 2 * GUARD,), float("nan"), dtype=torch.float16, device=dev)

    def view(self, out):
        return out[GUARD:-GUARD].view(self.shape)

    def _args(self, out):
        n, _, H, W = self.images.shape
        return c_api.EncoderArgs(self.images.data_ptr(), c_api.DBA_F16 if self.images.dtype == torch.float16 else c_api.DBA_F32, n, H, W,
                                 ctypes.pointer(self.wt), self.norm, self.od, self.view(out).data_ptr(), self.ws.data_ptr(), self.lay["total"],
                                 stream().value)

    def prefix(self, k):
        c_api.check(self.L.dba_encoder_forward_prefix(ctypes.byref(self._args(self.out)), k), "encoder_forward_prefix")
        torch.cuda.synchronize()

    def forward(self):
        out = self.new_out()
        c_api.check(self.L.dba_encoder_forward(ctypes.byref(self._args(out))), "encoder_forward")
        torch.cuda.synchronize()
        self.check_guards(out, "dba_encoder_forward")
        return self.view(out)

    def check_guards(self, out, what):
        fill = bits(torch.full((1,), float("nan"), dtype=torch.float16, device=dev))
        assert bool((bits(out[:GUARD]) == fill).all()) and bool((bits(out[-GUARD:]) == fill).all()), "%s wrote outside its output" % what
        assert bool((self.buf[self.lay["total"]:] == 255).all()), "%s wrote past its workspace" % what


@pytest.fixture(scope="module")
def gpu():
    """the card the reports name, read once"""
    return card()


def _report(gpu, case, name, per_kind):
    line = dict(case=case, encoder=name, gpu=gpu, **per_kind)
    print("ENC_STAGES " + json.dumps(line))
    path = os.environ.get("ENC_STAGES_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(line) + "\n")


def _kind(row):
    if row["kind"] != "conv":
        return row["kind"]
    return "conv_%s_K%d" % (row["epi"], 9 * row["src"][1] if row["ks"] == 3 else row["src"][1])


@pytest.mark.parametrize("name", ["fnet", "cnet"])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_every_launch_matches_fp64(capi, gpu, case, name):
    images = case_images(case)
    sd = case_weights(case, ENCODERS[name][0])
    run = Run(capi, name, sd, images)
    rows = stage_table(run.norm)
    assert len(rows) == run.lay["n_launches"]
    sdd = {k: v.to(dev) for k, v in sd.items()}
    cache, per_kind = {}, {}
    before, out_before = run.ws.clone(), run.out.clone()
    for k, row in enumerate(rows, 1):
        run.prefix(k)
        after, out_after = run.ws.clone(), run.out.clone()
        run.check_guards(run.out, "launch %d (%s)" % (k, row["name"]))
        st = check_stage(row, before, after, run.lay, sdd, images, run.view(out_before), run.view(out_after), cache)
        agg = per_kind.setdefault(_kind(row), {})
        for key, v in st.items():
            if key != "K":
                agg[key] = min(agg.get(key, 1.0), v) if key == "correct" else max(agg.get(key, 0.0), v)
        before, out_before = after, out_after
    full = run.forward()
    assert torch.equal(bits(full), bits(run.view(run.out))), "dba_encoder_forward differs from its own launches run as a prefix"
    assert not bool(torch.isnan(full).any())
    _report(gpu, case[0], name, {k: {a: float("%.3g" % b) for a, b in v.items()} for k, v in per_kind.items()})


def _oracle_nan(sd, images, norm):
    """which outputs of the fp64 oracle are NaN, on the fp16-rounded images (the cast the encoder applies on load)"""
    sd64 = {k: v.double() for k, v in sd.items()}
    with torch.no_grad():
        return torch.isnan(oenc.encoder_forward(sd64, images.half().double()[None], "instance" if norm else "none")[0])


@pytest.mark.parametrize("name", ["fnet", "cnet"])
@pytest.mark.parametrize("value", [float("nan"), 1e6], ids=["nan", "beyond_fp16"])
def test_non_finite_pixel_gives_the_oracles_nans(capi, name, value):
    """one NaN pixel (or one fp32 value that the fp16 cast turns into inf) in image 1 of 3: exactly the outputs that are NaN in the
    fp64 oracle are NaN, and images 0 and 2 keep the bits of a run without it"""
    norm, od = ENCODERS[name]
    sd = synth.make_encoder_weights(3, od)
    clean = torch.randn(3, 3, 240, 320, generator=torch.Generator().manual_seed(5))
    dirty = clean.clone()
    dirty[1, 1, 117, 203] = value
    want = _oracle_nan(sd, dirty, norm)
    assert bool(want[1].any()) and not bool(want[0].any()) and not bool(want[2].any())
    assert bool(want[1].all()) == bool(norm)                       # the instance norm spreads it over the image; without it, its neighbourhood
    ref = Run(capi, name, sd, clean).forward()
    got = Run(capi, name, sd, dirty).forward()
    assert torch.equal(torch.isnan(got).cpu(), want), "%d outputs differ from the oracle in being NaN" % int((torch.isnan(got).cpu() != want).sum())
    assert torch.equal(bits(got[0]), bits(ref[0])) and torch.equal(bits(got[2]), bits(ref[2]))
