"""Cost of prosody interpolation: the K = 2 mixed decode (MegaPLM.infer_mix) against infer on the stacked 2B rows (the
same encoder work) and on the B rows alone, at B = 1, 16, 64 with T = 64 and at the C3 shape (B = 16, T = 512); the mix
kernel's device time per launch (torch.profiler, launched without PDL); and a C4 synthesize (bench.py's workload, batch
64) with and without one prosody prompt.  Arms alternate within each round.  GPU only; prints JSON lines, the card's
name and power limit first.

    python tools/bench_prosody_mix.py [--rounds 3] [--skip-c3] [--skip-c4]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import helpers  # noqa: E402
from oracle import weights  # noqa: E402  (seeded weight specs only; nothing of the oracle is timed here)

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed_ms(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def kernel_us(K, B, V, reps=200):
    """Mean device time of one mix launch over `reps` launches."""
    from megatts2_b200 import _lib as L
    from megatts2_b200 import ops
    lib = L.lib()
    z = torch.randn(K * B, V, device=DEV) * 3
    w = torch.rand(B, K, device=DEV) + 0.1
    out = torch.empty(B, V, device=DEV)
    st = ops._stream()

    def launch():
        L.check(lib.mtts_mix_logprob_rows_f32(z.data_ptr(), V, V, K, B, w.data_ptr(), out.data_ptr(), V, st))

    from torch.profiler import ProfilerActivity, profile
    with ops.launch_policy(0, pdl=False):
        for _ in range(10):
            launch()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                launch()
            torch.cuda.synchronize()
    durs = [ev.time_range.elapsed_us() for ev in prof.events() if "mix_logprob_rows_kernel" in ev.name]
    if len(durs) != reps:
        raise RuntimeError(f"the profile holds {len(durs)} mix kernels, expected {reps}")
    return sum(durs) / reps


def decode_rounds(plm, B, T, rounds):
    g = torch.Generator().manual_seed(7 + B + T)
    tcs = [F.relu(torch.randn(B, T, 512, generator=g)).to(DEV) for _ in range(2)]
    stacked = torch.cat(tcs, 0)
    arms = {"mix_k2": lambda: plm.infer_mix(tcs, [0.5, 0.5]), "infer_2B": lambda: plm.infer(stacked),
            "infer_B": lambda: plm.infer(tcs[0])}
    for fn in arms.values():               # eager run + CUDA-graph capture of every arm before anything is timed
        for _ in range(3):
            fn()
    times = {n: [] for n in arms}
    for r in range(rounds):
        for name, fn in arms.items():
            times[name].append(timed_ms(fn))
    ref = times["infer_2B"]
    print(json.dumps({"B": B, "T": T, **{n + "_ms": [round(v, 2) for v in t] for n, t in times.items()},
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

    def step(prosody):
        mel = extract_mel_spec(wav, frames_major=True)
        kw = {}
        if prosody:
            kw = dict(prosody_mels=[extract_mel_spec(wav_p, frames_major=True)], prosody_weights=[0.5, 0.5])
        return tts.synthesize(phone, mel, forced_durations=forced, prompt_mels=mel, **kw)

    for p in (False, True):
        for _ in range(3):
            step(p)
    times = {"plain": [], "prosody": []}
    for r in range(rounds):
        for name, p in (("plain", False), ("prosody", True)):
            times[name].append(timed_ms(lambda: step(p)))
    print(json.dumps({"c4_B": bench.B_PER_GPU, **{n + "_ms": [round(v, 1) for v in t] for n, t in times.items()},
                      "prosody_vs_plain_pct": [round(100 * (a / b - 1), 2) for a, b in zip(times["prosody"],
                                                                                             times["plain"])]}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-c3", action="store_true")
    ap.add_argument("--skip-c4", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        sys.exit(1)
    print(json.dumps({"card": card()}), flush=True)
    for K, B in ((2, 1), (2, 16), (2, 64), (8, 64)):
        print(json.dumps({"mix_kernel_K": K, "B": B, "V": 1024, "us": round(kernel_us(K, B, 1024), 2)}), flush=True)
    t0 = time.time()
    plm = helpers.build_plm(weights.plm_state_dict(), DEV)
    print(json.dumps({"setup_s": round(time.time() - t0, 1)}), flush=True)
    for B in (1, 16, 64):
        decode_rounds(plm, B, 64, args.rounds)
    if not args.skip_c3:
        decode_rounds(plm, 16, 512, args.rounds)
    del plm
    torch.cuda.empty_cache()
    if not args.skip_c4:
        c4_rounds(args.rounds)


if __name__ == "__main__":
    main()
