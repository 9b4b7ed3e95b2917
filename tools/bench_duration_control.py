"""Cost of duration control: the pinned ADM decode (MegaADM.infer with pinned, a third of the phones pinned) against the
plain one at B = 1, 16, 64 with T = 64; fit_durations_kernel's device time per launch at B = 64 with Tp = 64 and 8192
(per-phone scale, pins and a total), from torch.profiler; and a C4 synthesize (bench.py's workload at batch 64, with the
ADM's durations instead of bench.py's forced ones) with total_frames = 1.25 x the ADM's totals, against the same call
without it.  Arms alternate within each round.  GPU only; prints JSON lines, the card's name, power limit and maximum SM
clock first.

    python tools/bench_duration_control.py [--rounds 3] [--skip-c4]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import helpers  # noqa: E402
from bench_prosody_mix import DEV, card, timed_ms  # noqa: E402
from oracle import weights  # noqa: E402  (seeded weight specs only; nothing of the oracle is timed here)


def pins(B, T, seed):
    r = np.random.default_rng(seed)
    return torch.from_numpy(np.where(r.random((B, T)) < 1 / 3, r.integers(1, 20, (B, T)), -1)).to(torch.int32)


def decode_rounds(adm, B, T, rounds):
    g = torch.Generator().manual_seed(7 + B)
    tc = F.relu(torch.randn(B, T, 512, generator=g)).to(DEV)
    p = pins(B, T, B).to(DEV)
    arms = {"plain": lambda: adm.infer(tc), "pinned": lambda: adm.infer(tc, pinned=p)}
    for fn in arms.values():               # eager run + CUDA-graph capture of every arm before anything is timed
        for _ in range(3):
            fn()
    times = {n: [] for n in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            times[name].append(timed_ms(fn))
    print(json.dumps({"B": B, "T": T, **{n + "_ms": [round(v, 3) for v in t] for n, t in times.items()},
                      "pinned_vs_plain_pct": [round(100 * (a / b - 1), 2) for a, b in zip(times["pinned"],
                                                                                          times["plain"])]}),
          flush=True)


def fit_us(B, Tp, reps=50):
    """Mean device time per launch of fit_durations_kernel over `reps` launches, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    from megatts2_b200 import ops
    g = torch.Generator().manual_seed(Tp)
    raw = (torch.rand(B, Tp, generator=g) * 12 + 0.5).to(DEV)
    scale = torch.rand(B, Tp, generator=g) + 0.5
    p = pins(B, Tp, Tp)
    free = (p < 1).sum(1)
    total = free + p.clamp(min=0).sum(1) + (free * 9)
    args = (scale.to(DEV), total.to(torch.int32), p)
    ops.fit_durations(raw, *args)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ops.fit_durations(raw, *args)
        torch.cuda.synchronize()
    durs = [ev.time_range.elapsed_us() for ev in prof.events() if "fit_durations_kernel" in ev.name]
    if len(durs) != reps:
        raise RuntimeError(f"the profile holds {len(durs)} fit_durations_kernel launches, expected {reps}")
    print(json.dumps({"fit_B": B, "Tp": Tp, "fit_us": round(sum(durs) / reps, 2)}), flush=True)


def c4_rounds(rounds):
    import bench
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    dev = torch.device(DEV)
    tts = bench.build_product(dev)
    wav, phone, _ = bench.make_inputs(range(bench.B_PER_GPU))
    wav, phone = wav.to(dev), phone.to(dev)
    mel0 = extract_mel_spec(wav, frames_major=True)
    adm_totals = tts.synthesize(phone, mel0, return_intermediates=True)["totals"]
    total = [int(round(1.25 * t)) for t in adm_totals]

    def step(fit):
        mel = extract_mel_spec(wav, frames_major=True)
        return tts.synthesize(phone, mel, prompt_mels=mel, **(dict(total_frames=total) if fit else {}))

    for fit in (False, True):
        for _ in range(3):
            step(fit)
    times = {"adm": [], "total_frames": []}
    for _ in range(rounds):
        for name, fit in (("adm", False), ("total_frames", True)):
            times[name].append(timed_ms(lambda: step(fit)))
    print(json.dumps({"c4_B": bench.B_PER_GPU, "adm_frames": sum(adm_totals), "fitted_frames": sum(total),
                      **{n + "_ms": [round(v, 1) for v in t] for n, t in times.items()},
                      "total_frames_vs_adm_pct": [round(100 * (a / b - 1), 2) for a, b in zip(
                          times["total_frames"], times["adm"])]}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-c4", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        sys.exit(1)
    print(json.dumps({"card": card()}), flush=True)
    t0 = time.time()
    adm = helpers.build_adm(weights.adm_state_dict(), DEV)
    print(json.dumps({"setup_s": round(time.time() - t0, 1)}), flush=True)
    for B in (1, 16, 64):
        decode_rounds(adm, B, 64, args.rounds)
    for Tp in (64, 8192):
        fit_us(64, Tp)
    del adm
    torch.cuda.empty_cache()
    if not args.skip_c4:
        c4_rounds(args.rounds)


if __name__ == "__main__":
    main()
