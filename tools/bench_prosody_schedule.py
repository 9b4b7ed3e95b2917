"""Cost of mix schedules (weights that change along the utterance): MegaPLM.infer_mix and MegaADM.infer_mix at K = 2,
T = 64, B = 1, 16, 64, with a (B, T, K) schedule against (B, K) weights; the phone -> step expansion kernel's device time
per launch (torch.profiler over many launches, at bench.py's C4 shape: B = 64, Tp = 64 phones of 8 frames, T = 64); and a
C4 synthesize (bench.py's workload, batch 64) with one prosody prompt, with per-phone weights against constant ones.
Arms alternate within each round.  GPU only; prints JSON lines, the card's name, power limit and maximum SM clock first.

    python tools/bench_prosody_schedule.py [--rounds 3] [--skip-c4]
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import helpers  # noqa: E402
from bench_prosody_mix import DEV, card, timed_ms  # noqa: E402
from oracle import weights  # noqa: E402  (seeded weight specs only; nothing of the oracle is timed here)


def latents(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return [F.relu(torch.randn(B, T, 512, generator=g)).to(DEV) for _ in range(2)]


def schedule(B, T, seed):
    """A glide from source 0 to source 1 along the utterance, with a per-utterance offset."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.linspace(0, 1, T)[None, :] + 0.2 * torch.rand(B, 1, generator=g)).clamp(0, 1)
    return torch.stack([1 - x + 0.01, x], -1)


def decode_rounds(name, fn, B, T, rounds):
    tcs = latents(B, T, 7 + B + T)
    sched = schedule(B, T, B)
    rows = sched.mean(1)
    arms = {"rows": lambda: fn(tcs, rows), "schedule": lambda: fn(tcs, sched)}
    for f in arms.values():                # eager run + CUDA-graph capture of every arm before anything is timed
        for _ in range(3):
            f()
    times = {n: [] for n in arms}
    for _ in range(rounds):
        for n, f in arms.items():
            times[n].append(timed_ms(f))
    print(json.dumps({"model": name, "K": 2, "B": B, "T": T, **{n + "_ms": [round(v, 3) for v in t] for n, t in times.items()},
                      "schedule_vs_rows_pct": [round(100 * (a / b - 1), 2) for a, b in zip(times["schedule"],
                                                                                           times["rows"])]}), flush=True)


def expansion_us(rounds, reps=200):
    """Mean device time per launch of mix_step_weights_kernel, from torch.profiler over `reps` launches per round."""
    from torch.profiler import ProfilerActivity, profile
    from megatts2_b200 import ops
    B, Tp = 64, 64
    pw = torch.rand(B, Tp, 2, device=DEV) + 0.01
    d = torch.full((B, Tp), 8, dtype=torch.int32, device=DEV)
    for _ in range(10):
        ops.mix_step_weights(pw, d, Tp)
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                ops.mix_step_weights(pw, d, Tp)
            torch.cuda.synchronize()
        durs = [ev.time_range.elapsed_us() for ev in prof.events() if "mix_step_weights_kernel" in ev.name]
        if len(durs) != reps:
            raise RuntimeError(f"the profile holds {len(durs)} mix_step_weights_kernel launches, expected {reps}")
        out.append(sum(durs) / reps)
    print(json.dumps({"expansion_B": B, "Tp": Tp, "T": Tp, "K": 2, "us_per_launch": [round(v, 2) for v in out]}),
          flush=True)


def c4_rounds(rounds):
    import bench
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    dev = torch.device(DEV)
    tts = bench.build_product(dev)
    wav, phone, forced = bench.make_inputs(range(bench.B_PER_GPU))
    wav_p, _, _ = bench.make_inputs(range(1000, 1000 + bench.B_PER_GPU))     # other utterances' audio: the prosody prompts
    wav, phone, forced, wav_p = wav.to(dev), phone.to(dev), forced.to(dev), wav_p.to(dev)
    B, Tp = phone.shape
    per_phone = schedule(B, Tp, 3)

    def step(w):
        mel = extract_mel_spec(wav, frames_major=True)
        return tts.synthesize(phone, mel, forced_durations=forced, prompt_mels=mel,
                              prosody_mels=[extract_mel_spec(wav_p, frames_major=True)], prosody_weights=w)

    arms = {"constant": [0.5, 0.5], "per_phone": per_phone}
    for w in arms.values():
        for _ in range(3):
            step(w)
    times = {n: [] for n in arms}
    for _ in range(rounds):
        for n, w in arms.items():
            times[n].append(timed_ms(lambda: step(w)))
    print(json.dumps({"c4_B": B, "Tp": Tp, **{n + "_ms": [round(v, 1) for v in t] for n, t in times.items()},
                      "per_phone_vs_constant_pct": [round(100 * (a / b - 1), 2) for a, b in zip(
                          times["per_phone"], times["constant"])]}), flush=True)


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
    plm = helpers.build_plm(weights.plm_state_dict(), DEV)
    adm = helpers.build_adm(weights.adm_state_dict(), DEV)
    print(json.dumps({"setup_s": round(time.time() - t0, 1)}), flush=True)
    expansion_us(args.rounds)
    for B in (1, 16, 64):
        decode_rounds("plm", plm.infer_mix, B, 64, args.rounds)
        decode_rounds("adm", adm.infer_mix, B, 64, args.rounds)
    del plm, adm
    torch.cuda.empty_cache()
    if not args.skip_c4:
        c4_rounds(args.rounds)


if __name__ == "__main__":
    main()
