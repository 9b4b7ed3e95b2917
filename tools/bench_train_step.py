"""Time one PLM training step with its dense products on bf16x3 operands (the training format) against f16x2 operands
(what training used before: 3 MMAs per product instead of 6, but tiny gradients flush to zero), in one process,
alternating the two (GPU only).

A step is MegaPLM.forward in train mode (seeded weights, dropout on) + cross-entropy + backward + AdamW, at B x T tokens.
Prints one JSON line: per-format step times of every round, and the card they were measured on.

    python tools/bench_train_step.py [--batch 8] [--frames 320] [--rounds 3] [--steps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import helpers  # noqa: E402
from megatts2_b200 import autograd, pack  # noqa: E402
from oracle import weights  # noqa: E402

FORMATS = (("bf16x3", pack.FMT_BF16X3), ("f16x2", pack.FMT_F16X2))


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--frames", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = "cuda"
    plm = helpers.build_plm(weights.plm_state_dict(), dev)
    plm.train()
    opt = torch.optim.AdamW(plm.parameters(), lr=1e-6)
    g = torch.Generator().manual_seed(3)
    B, T = a.batch, a.frames
    tc = F.relu(torch.randn(B, T, 512, generator=g)).to(dev)
    codes = torch.cat([torch.full((B, 1), 1024), torch.randint(0, 1024, (B, T), generator=g)], 1).to(dev)
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)

    def step():
        opt.zero_grad(set_to_none=True)
        logits, y = plm(tc, codes, lens)
        F.cross_entropy(logits.float().transpose(1, 2), y, ignore_index=1025).backward()
        opt.step()

    def timed(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            step()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    res = {name: [] for name, _ in FORMATS}
    with pack.engine_scope(pack.ENGINE_F16X2):
        for r in range(a.rounds):
            for name, fmt in FORMATS:
                autograd._train_fmt = lambda fmt=fmt: fmt
                if r == 0:
                    timed(2)                       # warm-up: module loads, TMA descriptors, allocator
                res[name].append(round(timed(a.steps), 2))
    print(json.dumps({"workload": f"PLM training step (forward + backward + AdamW), {B} x {T} tokens, engine f16x2",
                      "step_ms": res, "card": card()}))


if __name__ == "__main__":
    main()
