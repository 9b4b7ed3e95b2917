"""The fused ResBlock kernel (resblock_tc.cu) against the two-launch tap-GEMM flow it replaces.

MEGATTS2_RB_FUSE is read once per process, so each side runs in a subprocess; the waveforms must be bit-identical, the
fused side must issue fewer launches (the C <= 64 stages took the new path), and the fp16 range flag must be raised
exactly when the unfused flow raises it."""
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
for name, (cfg, B, T, engine, w1_scale, up_scale) in cases.items():
    if cfg is None:
        h = helpers.build_hifigan(weights.hifigan_state_dict(), "cuda")
    else:
        gen = HifiganGenerator(**cfg)
        with torch.no_grad():
            for p in gen.parameters():
                p.copy_(torch.randn_like(p) * (0.5 / p[0].numel() ** 0.5) if p.dim() > 1 else torch.randn_like(p) * 0.1)
            for rb in gen.resblocks:
                for c in rb.convs1:
                    c.weight.mul_(w1_scale)
            gen.ups[0].weight.mul_(up_scale)
        h = HIFIGAN(gen.to(dev)).eval()
    h.generator.engine = engine
    mel = (torch.randn(B, T, 80, generator=torch.Generator().manual_seed(B * 1000 + T)) * 2 - 4).to(dev)
    ops.tc_overflow(dev)                       # clear the flag
    n0 = ops.launch_count()
    wav = h.decode_batch_cl(mel)
    torch.cuda.synchronize()
    out[name] = (wav.cpu(), ops.tc_overflow(dev), ops.launch_count() - n0)
torch.save(out, {path!r})
"""

# two stages, C = 64 (L = 2 (T + 10)) and C = 32 (L = 4 (T + 10))
_SMALL = dict(upsample_initial_channel=128, upsample_factors=(2, 2), upsample_kernel_sizes=(4, 4))
# k = 3 at dilation 30: h1 + h2 = 31, so the C = 64 stage of a 6-frame mel (L = 32) is the shortest sequence accepted
_MIN = dict(_SMALL, resblock_kernel_sizes=(3, 11), resblock_dilation_sizes=((1, 30, 2), (1, 3, 5)))

CASES = {}
for _e, _en in ((2, "f16x2"), (3, "f16")):
    CASES.update({
        f"v1_b1_{_en}": (None, 1, 8, _e, 1.0, 1.0),                     # HiFi-GAN V1: C = 64 at L = 2304, C = 32 at L = 4608
        f"partial_b3_{_en}": (_SMALL, 3, 90, _e, 1.0, 1.0),            # L = 200 / 400: several tiles, the last one partial
        f"partial_b1_{_en}": (_SMALL, 1, 90, _e, 1.0, 1.0),
        f"one_tile_b3_{_en}": (_SMALL, 3, 40, _e, 1.0, 1.0),           # L = 100 at C = 64: shorter than one tile, both ends reflect
        f"shortest_b4_{_en}": (_MIN, 4, 6, _e, 1.0, 1.0),              # L = 32 = h1 + h2 + 1 at C = 64
        f"overflow_b3_{_en}": (_SMALL, 3, 40, _e, 3.0e4, 1.0),    # conv1 outputs beyond the fp16 range
        f"overflow_x_b3_{_en}": (_SMALL, 3, 40, _e, 1.0, 1.0e6),  # the C = 64 stage's input x beyond the fp16 range
    })


def _run(fuse, tmp_path):
    path = str(tmp_path / f"rb{fuse}.pt")
    src = _SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, "tests"), path=path, cases=CASES)
    subprocess.run([sys.executable, "-c", src], check=True, env=dict(os.environ, MEGATTS2_RB_FUSE=fuse), cwd=ROOT,
                   timeout=600)
    return torch.load(path)


@gpu
@pytest.mark.timeout(900)
def test_fused_resblock_is_bit_identical_to_two_launch_flow(tmp_path):
    fused, plain = _run("1", tmp_path), _run("0", tmp_path)
    for name in CASES:
        (wf, of, nf), (wp, op, np_) = fused[name], plain[name]
        assert nf < np_, f"{name}: the fused path did not run ({nf} vs {np_} launches)"
        assert of == op, f"{name}: fp16 range flag {of} (fused) vs {op} (two launches)"
        assert torch.equal(torch.isnan(wf), torch.isnan(wp)), name
        assert torch.equal(torch.nan_to_num(wf), torch.nan_to_num(wp)), f"{name}: max diff {(wf - wp).abs().max().item()}"
        if name.startswith("overflow"):
            assert of, f"{name}: the flag should be raised"
        else:
            assert not of and bool(torch.isfinite(wf).all()), name
