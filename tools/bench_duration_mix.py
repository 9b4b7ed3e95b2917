"""Cost of duration interpolation: the K = 2 mixed ADM decode (MegaADM.infer_mix) against infer on the stacked 2B rows
(the same encoder work) and on the B rows alone, at B = 1, 16, 64 with T = 64; the readout kernels' device time per
launch, adm_readout_mix_kernel (K = 2) against adm_readout_kernel on the same 2B rows, taken from torch.profiler over
whole eager decodes launched without PDL; and a C4 synthesize (bench.py's workload, batch 64) with one prosody prompt,
with and without duration_weights.  Arms alternate within each round.  GPU only; prints JSON lines, the card's name,
power limit and maximum SM clock first.

    python tools/bench_duration_mix.py [--rounds 3] [--skip-c4]
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


def readout_us(adm, B, T):
    """Mean device time per launch of each readout kernel over one eager decode each (T launches)."""
    from torch.profiler import ProfilerActivity, profile
    from megatts2_b200 import graphs, ops
    tcs = latents(B, T, 11 + B)
    stacked = torch.cat(tcs, 0)
    with graphs.disabled(), ops.launch_policy(0, pdl=False):
        adm.infer_mix(tcs, [0.5, 0.5])
        adm.infer(stacked)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            adm.infer_mix(tcs, [0.5, 0.5])
            adm.infer(stacked)
            torch.cuda.synchronize()
    out = {}
    for name in ("adm_readout_mix_kernel", "adm_readout_kernel"):
        durs = [ev.time_range.elapsed_us() for ev in prof.events() if name in ev.name]
        if len(durs) != T:
            raise RuntimeError(f"the profile holds {len(durs)} {name} launches, expected {T}")
        out[name + "_us"] = round(sum(durs) / T, 2)
    print(json.dumps({"readout_B": B, "K": 2, "T": T, **out}), flush=True)


def decode_rounds(adm, B, T, rounds):
    tcs = latents(B, T, 7 + B + T)
    stacked = torch.cat(tcs, 0)
    arms = {"mix_k2": lambda: adm.infer_mix(tcs, [0.5, 0.5]), "infer_2B": lambda: adm.infer(stacked),
            "infer_B": lambda: adm.infer(tcs[0])}
    for fn in arms.values():               # eager run + CUDA-graph capture of every arm before anything is timed
        for _ in range(3):
            fn()
    times = {n: [] for n in arms}
    for r in range(rounds):
        for name, fn in arms.items():
            times[name].append(timed_ms(fn))
    ref = times["infer_2B"]
    print(json.dumps({"B": B, "T": T, **{n + "_ms": [round(v, 3) for v in t] for n, t in times.items()},
                      "mix_vs_infer_2B_pct": [round(100 * (a / b - 1), 2) for a, b in zip(times["mix_k2"], ref)],
                      "mix_vs_infer_B_pct": [round(100 * (a / b - 1), 2) for a, b in zip(times["mix_k2"], times["infer_B"])]}),
          flush=True)


def c4_rounds(rounds):
    import bench
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    dev = torch.device(DEV)
    tts = bench.build_product(dev)
    wav, phone, forced = bench.make_inputs(range(bench.B_PER_GPU))
    wav_p, _, _ = bench.make_inputs(range(1000, 1000 + bench.B_PER_GPU))     # other utterances' audio: the prosody prompts
    wav, phone, forced, wav_p = wav.to(dev), phone.to(dev), forced.to(dev), wav_p.to(dev)

    def step(durations):
        mel = extract_mel_spec(wav, frames_major=True)
        kw = dict(prosody_mels=[extract_mel_spec(wav_p, frames_major=True)], prosody_weights=[0.5, 0.5])
        if durations:
            kw["duration_weights"] = [0.5, 0.5]
        return tts.synthesize(phone, mel, forced_durations=forced, prompt_mels=mel, **kw)

    for d in (False, True):
        for _ in range(3):
            step(d)
    times = {"prosody": [], "prosody_durations": []}
    for r in range(rounds):
        for name, d in (("prosody", False), ("prosody_durations", True)):
            times[name].append(timed_ms(lambda: step(d)))
    print(json.dumps({"c4_B": bench.B_PER_GPU, **{n + "_ms": [round(v, 1) for v in t] for n, t in times.items()},
                      "durations_vs_prosody_pct": [round(100 * (a / b - 1), 2) for a, b in zip(
                          times["prosody_durations"], times["prosody"])]}),
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
    for B in (1, 64):
        readout_us(adm, B, 32)
    for B in (1, 16, 64):
        decode_rounds(adm, B, 64, args.rounds)
    del adm
    torch.cuda.empty_cache()
    if not args.skip_c4:
        c4_rounds(args.rounds)


if __name__ == "__main__":
    main()
