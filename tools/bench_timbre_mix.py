"""Cost of timbre interpolation on bench.py's utterance shapes (Tp = 64 phones, Tm = 500 prompt frames):
MRTE.tc_latent_mix at K = 2 against two tc_latent calls and against one, at B = 1, 16, 64; a C4 synthesize (bench.py's
workload, batch 64) with one timbre prompt against without; and a C4 synthesize with one prosody prompt, whose prompt
latent now comes from the call's single phone-encoder pass.  Arms alternate within each round.  With --profile, the
device time per launch of mix_layernorm_kernel (K = 2 and K = 8) against layernorm_reg_kernel on the same rows, from
torch.profiler in a run of its own.  GPU only; prints JSON lines, the card's name, power limit and maximum SM clock first.

    python tools/bench_timbre_mix.py [--rounds 3] [--skip-c4]
    python tools/bench_timbre_mix.py --profile
    python tools/bench_timbre_mix.py --c4-only plain,prosody      (also runs on a tree without timbre_mels)
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import helpers  # noqa: E402
from bench_prosody_mix import DEV, card, timed_ms  # noqa: E402
from oracle import weights  # noqa: E402  (seeded weight specs only; nothing of the oracle is timed here)

TP, TM = 64, 500


def mrte_inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    phone = torch.randint(0, 320, (B, TP), generator=g).to(DEV)
    mels = [(torch.randn(B, TM, 80, generator=g) * 2 - 4).to(DEV) for _ in range(2)]
    return phone, mels


def mrte_rounds(mrte, B, rounds):
    phone, mels = mrte_inputs(B, 5 + B)
    with torch.no_grad():
        arms = {"mix_k2": lambda: mrte.tc_latent_mix(phone, mels, [0.5, 0.5]),
                "tc_latent_x2": lambda: [mrte.tc_latent(phone, m) for m in mels],
                "tc_latent_x1": lambda: mrte.tc_latent(phone, mels[0])}
        for fn in arms.values():
            for _ in range(3):
                fn()
        times = {n: [] for n in arms}
        for _ in range(rounds):
            for name, fn in arms.items():
                times[name].append(timed_ms(fn))
    print(json.dumps({"mrte_B": B, "Tp": TP, "Tm": TM, **{n + "_ms": [round(v, 3) for v in t] for n, t in times.items()},
                      "mix_vs_x2_pct": [round(100 * (a / b - 1), 2) for a, b in zip(times["mix_k2"], times["tc_latent_x2"])]}),
          flush=True)


def kernel_us(B, reps=50):
    """Mean device time per launch of mix_layernorm_kernel<4> (K = 2, 8) and layernorm_reg_kernel<4> on B * Tp rows of
    512, from torch.profiler, launched without PDL."""
    from torch.profiler import ProfilerActivity, profile
    from megatts2_b200 import _lib as L
    from megatts2_b200 import ops
    g = torch.Generator().manual_seed(B)
    ys = torch.randn(8, B, TP, 512, generator=g).to(DEV)
    gamma, beta = torch.ones(512, device=DEV), torch.zeros(512, device=DEV)
    w2, w8 = torch.tensor([0.5, 0.5], device=DEV), torch.full((8,), 0.125, device=DEV)
    out = torch.empty(B, TP, 512, device=DEV)
    arms = {"mix_k2": (lambda: ops.mix_layernorm(ys[:2], w2, gamma, beta, post_act=L.ACT_RELU, out=out),
                       "mix_layernorm_kernel"),
            "mix_k8": (lambda: ops.mix_layernorm(ys, w8, gamma, beta, post_act=L.ACT_RELU, out=out),
                       "mix_layernorm_kernel"),
            "layernorm": (lambda: ops.layernorm(ys[0], gamma, beta, post_act=L.ACT_RELU, out=out), "layernorm_reg_kernel")}
    res = {}
    with ops.launch_policy(0, pdl=False):
        for name, (fn, kernel) in arms.items():
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    fn()
                torch.cuda.synchronize()
            durs = [ev.time_range.elapsed_us() for ev in prof.events() if kernel in ev.name]
            if len(durs) < reps - 2:               # the trace may drop a launch at its edge; never more than that
                raise RuntimeError(f"the profile holds {len(durs)} {kernel} launches, expected {reps}")
            res[name + "_us"] = round(sum(durs) / len(durs), 2)
    print(json.dumps({"kernel_B": B, "rows": B * TP, "C": 512, **res}), flush=True)


def c4_rounds(rounds, arms):
    import bench
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    dev = torch.device(DEV)
    tts = bench.build_product(dev)
    wav, phone, forced = bench.make_inputs(range(bench.B_PER_GPU))
    wav_p, _, _ = bench.make_inputs(range(1000, 1000 + bench.B_PER_GPU))     # other utterances' audio: the prompts
    wav, phone, forced, wav_p = wav.to(dev), phone.to(dev), forced.to(dev), wav_p.to(dev)

    def step(arm):
        mel = extract_mel_spec(wav, frames_major=True)
        kw = {}
        if arm == "timbre":
            kw = dict(timbre_mels=[extract_mel_spec(wav_p, frames_major=True)], timbre_weights=[0.5, 0.5])
        elif arm == "prosody":
            kw = dict(prosody_mels=[extract_mel_spec(wav_p, frames_major=True)], prosody_weights=[0.5, 0.5])
        return tts.synthesize(phone, mel, forced_durations=forced, prompt_mels=mel, **kw)

    for a in arms:
        for _ in range(3):
            step(a)
    times = {a: [] for a in arms}
    for _ in range(rounds):
        for a in arms:
            times[a].append(timed_ms(lambda: step(a)))
    pct = {}
    if "timbre" in times:
        pct["timbre_vs_plain_pct"] = [round(100 * (a / b - 1), 2) for a, b in zip(times["timbre"], times["plain"])]
    print(json.dumps({"c4_B": bench.B_PER_GPU, **{n + "_ms": [round(v, 1) for v in t] for n, t in times.items()}, **pct}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-c4", action="store_true")
    ap.add_argument("--profile", action="store_true", help="only the per-launch kernel times (torch.profiler)")
    ap.add_argument("--c4-only", default=None, metavar="ARMS",
                    help="only the C4 rounds of these comma-separated arms (plain, timbre, prosody)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        sys.exit(1)
    print(json.dumps({"card": card()}), flush=True)
    if args.profile:
        for B in (1, 16, 64):
            kernel_us(B)
        return
    if args.c4_only:
        c4_rounds(args.rounds, args.c4_only.split(","))
        return
    t0 = time.time()
    g = helpers.build_g(weights.g_state_dict(), DEV)
    print(json.dumps({"setup_s": round(time.time() - t0, 1)}), flush=True)
    for B in (1, 16, 64):
        mrte_rounds(g.mrte, B, args.rounds)
    del g
    torch.cuda.empty_cache()
    if not args.skip_c4:
        c4_rounds(args.rounds, ("plain", "timbre", "prosody"))


if __name__ == "__main__":
    main()
