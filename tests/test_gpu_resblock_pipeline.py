"""The fused ResBlock kernel (resblock_tc.cu) with many work items per CTA, against the two-launch tap-GEMM flow.

The loader warps fill a ring of x buffers ahead of the consumer warpgroups, handing each buffer over through the
xfull / xempty mbarriers.  At full grid width a CTA takes about one item, so the ring never wraps; here the persistent
grids are limited to 1, 2 and 3 SMs, so each warpgroup takes tens of items and every buffer and barrier parity is
reused many times, with even and odd item counts per CTA (an odd count leaves warpgroup 1 without a last item).
MEGATTS2_RB_FUSE is read once per process, so each side runs in a subprocess; the waveforms must be bit-identical and
the fp16 range flag must match."""
import os
import subprocess
import sys

import pytest
import torch

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCRIPT = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import helpers
from megatts2_b200 import ops
from megatts2_b200.models.megatts2 import HIFIGAN, HifiganGenerator
from oracle import weights
torch.manual_seed(0)
cases = {cases!r}
out = {{}}
dev = torch.device("cuda", 0)
for name, (cfg, B, T, engine, up_scale) in cases.items():
    if cfg is None:
        h = helpers.build_hifigan(weights.hifigan_state_dict(), "cuda")
    else:
        gen = HifiganGenerator(**cfg)
        with torch.no_grad():
            for p in gen.parameters():
                p.copy_(torch.randn_like(p) * (0.5 / p[0].numel() ** 0.5) if p.dim() > 1 else torch.randn_like(p) * 0.1)
            gen.ups[0].weight.mul_(up_scale)
        h = HIFIGAN(gen.to(dev)).eval()
    h.generator.engine = engine
    mel = (torch.randn(B, T, 80, generator=torch.Generator().manual_seed(B * 1000 + T)) * 2 - 4).to(dev)
    for sms in {sms!r}:
        ops.tc_overflow(dev)                   # clear the flag
        n0 = ops.launch_count()
        with ops.launch_policy(sms):
            wav = h.decode_batch_cl(mel)
        torch.cuda.synchronize()
        out[(name, sms)] = (wav.cpu(), ops.tc_overflow(dev), ops.launch_count() - n0)
torch.save(out, {path!r})
"""

SMS = (1, 2, 3)
# two stages: C = 64 at L = 2 (T + 10), C = 32 at L = 4 (T + 10); kernel sizes 3, 7, 11 at dilations 1, 3, 5
_SMALL = dict(upsample_initial_channel=128, upsample_factors=(2, 2), upsample_kernel_sizes=(4, 4))

CASES = {}
for _e, _en in ((2, "f16x2"), (3, "f16")):
    CASES.update({
        # HiFi-GAN V1: C = 64 at L = 2304 (38-40 items per step), C = 32 at L = 4608 (74-80 items per step)
        f"v1_b2_{_en}": (None, 2, 8, _e, 1.0),
        # C = 64 at L = 350: 3 tiles of each item at every k, 9 items per step (odd on 1 and 3 SMs)
        f"odd_b3_{_en}": (_SMALL, 3, 165, _e, 1.0),
    })
# the C = 64 stage's input x beyond the fp16 range: the loader raises the flag
CASES["odd_overflow_x_b3_f16x2"] = (_SMALL, 3, 165, 2, 1.0e6)


def _run(fuse, tmp_path):
    path = str(tmp_path / f"rbp{fuse}.pt")
    src = _SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, "tests"), path=path, cases=CASES, sms=SMS)
    subprocess.run([sys.executable, "-c", src], check=True, env=dict(os.environ, MEGATTS2_RB_FUSE=fuse), cwd=ROOT,
                   timeout=600)
    return torch.load(path)


@gpu
@pytest.mark.timeout(900)
def test_fused_resblock_many_items_per_cta_is_bit_identical(tmp_path):
    fused, plain = _run("1", tmp_path), _run("0", tmp_path)
    for name in CASES:
        for sms in SMS:
            key = f"{name} on {sms} SMs"
            (wf, of, nf), (wp, op, np_) = fused[(name, sms)], plain[(name, sms)]
            assert nf < np_, f"{key}: the fused path did not run ({nf} vs {np_} launches)"
            assert of == op, f"{key}: fp16 range flag {of} (fused) vs {op} (two launches)"
            assert torch.equal(torch.isnan(wf), torch.isnan(wp)), key
            assert torch.equal(torch.nan_to_num(wf), torch.nan_to_num(wp)), f"{key}: max diff {(wf - wp).abs().max().item()}"
            if "overflow" in name:
                assert of, f"{key}: the flag should be raised"
            else:
                assert not of and bool(torch.isfinite(wf).all()), key
