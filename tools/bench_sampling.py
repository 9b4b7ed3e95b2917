"""Cost of the opt-in sampled PLM decode: the C3 decode (MegaPLM.infer, B = 16, T = 512) greedy against sampled (no
filter, top-k 50, top-p 0.9), in alternated rounds, and the sampler kernel's device time per launch (torch.profiler,
launched without PDL) at B = 16 and 64.  GPU only; prints JSON lines, the card's name and power limit first.

    python tools/bench_sampling.py [--rounds 3] [--B 16] [--T 512]
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
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def kernel_us(B, V, sampling, reps=200):
    """Mean device time of one sampler launch (and of the greedy argmax launch, for comparison) over `reps` launches."""
    from megatts2_b200 import _lib as L
    from megatts2_b200 import ops
    lib = L.lib()
    z = torch.randn(B, V, device=DEV) * 3
    seed, keys = sampling.seed_tensor(z.device), torch.arange(B, dtype=torch.int64, device=DEV)
    out = torch.empty(B, dtype=torch.int64, device=DEV)
    s = sampling.struct(seed, keys)
    st = ops._stream()

    def launch():
        L.check(lib.mtts_sample_rows_f32(z.data_ptr(), V, V, B, 7, C.byref(s), out.data_ptr(), 1, st))

    from torch.profiler import ProfilerActivity, profile
    # without programmatic dependent launch: with it, a back-to-back launch becomes resident while its predecessor runs,
    # and its span would include that wait
    with ops.launch_policy(0, pdl=False):
        for _ in range(10):
            launch()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                launch()
            torch.cuda.synchronize()
    durs = [ev.time_range.elapsed_us() for ev in prof.events()
            if "sample_rows_kernel" in ev.name or "argmax_rows_kernel" in ev.name]
    if len(durs) != reps:
        raise RuntimeError(f"the profile holds {len(durs)} sampler kernels, expected {reps}")
    return sum(durs) / reps, reps


def decode_rounds(args):
    from megatts2_b200.sampling import Sampling
    t0 = time.time()
    plm = helpers.build_plm(weights.plm_state_dict(), DEV)
    tc = F.relu(torch.randn(args.B, args.T, 512, generator=torch.Generator().manual_seed(7))).to(DEV)
    modes = {"greedy": None, "sampled": Sampling(temperature=1.0, seed=1), "top_k50": Sampling(top_k=50, seed=1),
             "top_p0.9": Sampling(top_p=0.9, seed=1)}
    for name, s in modes.items():         # eager run + CUDA-graph capture of every mode before anything is timed
        for _ in range(2):
            plm.infer(tc, sampling=s)
    torch.cuda.synchronize()
    print(json.dumps({"setup_s": round(time.time() - t0, 1)}), flush=True)
    times = {n: [] for n in modes}
    for r in range(args.rounds):
        for name, s in modes.items():
            ms, _ = timed_ms(lambda: plm.infer(tc, sampling=s))
            times[name].append(ms)
            print(json.dumps({"round": r, "mode": name, "decode_ms": round(ms, 1)}), flush=True)
    g = times["greedy"]
    for name in modes:
        print(json.dumps({"mode": name, "B": args.B, "T": args.T, "decode_ms": [round(v, 1) for v in times[name]],
                          "vs_greedy_pct": [round(100 * (v / b - 1), 2) for v, b in zip(times[name], g)]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternated decode rounds (0: only the kernel times)")
    ap.add_argument("--B", type=int, default=16)
    ap.add_argument("--T", type=int, default=512)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        sys.exit(1)
    from megatts2_b200.sampling import Sampling
    print(json.dumps({"card": card()}), flush=True)
    if args.rounds > 0:
        decode_rounds(args)
    for B in (16, 64):
        row = {"kernel_B": B}
        for name, s in (("argmax", Sampling(top_k=1)), ("sampled", Sampling()), ("top_k50", Sampling(top_k=50)),
                        ("top_p0.9", Sampling(top_p=0.9))):
            us, n = kernel_us(B, 1024, s)
            row[name + "_us"] = round(us, 2)
        row["steps_per_decode"] = args.T
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
