"""The f16 inference engine against the default f16x2 engine, in one process, alternating f16x2 / f16 (GPU only).

Two workloads, as bench.py defines them: the C4 step (batch 64 full synthesis with the prompt re-vocode, a 256 MiB L2
flush before every timed step) and the C3 PLM decode (512 prosody tokens, batch 16).  Each round times both workloads
under f16x2, then under f16; rounds repeat --rounds times, so every f16 number has an f16x2 neighbour measured minutes
apart on the same card.  Then one eager step / decode per engine runs inside the library's tap-GEMM profile
(mtts_profile_begin / end: CUDA events around every tap-GEMM launch) for the tap-GEMM time, algorithmic TFLOP and launch
count.  Prints one JSON line per engine; the f16 line also carries its outputs against the f16x2 run of the same inputs.

    python tools/bench_engines.py [--rounds 3] [--steps 3] [--decodes 1]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from megatts2_b200 import _lib as L, graphs, pack  # noqa: E402

ENGINES = (("f16x2", pack.ENGINE_F16X2, 3), ("f16", pack.ENGINE_F16, 1))     # (name, engine, MMAs per product)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:            # the numbers below still stand; the card is then named by torch only
        out = f"nvidia-smi unavailable: {e}"
    return {"nvidia_smi": dict(zip(q.split(","), [c.strip() for c in out.split(",")])) if "," in out else out,
            "torch_name": torch.cuda.get_device_name(0)}


def timed(fn, n, flush=None):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        if flush is not None:
            flush.zero_()
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, out


def profile(fn):
    """tap-GEMM ms, TFLOP and launches of one eager call (wgmma launches incl. their activation-split kernels)"""
    lib = L.lib()
    lib.mtts_profile_begin()
    with graphs.disabled():
        fn()
    ms, fl, n = C.c_double(), C.c_double(), C.c_int64()
    L.check(lib.mtts_profile_end(C.byref(ms), C.byref(fl), C.byref(n)))
    sp = (C.c_double * 6)()
    lib.mtts_profile_split(sp)
    return {"tc_ms": sp[3], "tc_tflop": sp[4] / 1e12, "tc_launches": int(sp[5]),
            "ffma_ms": sp[0], "ffma_tflop": sp[1] / 1e12, "ffma_launches": int(sp[2])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3, help="timed C4 steps per engine and round")
    ap.add_argument("--decodes", type=int, default=1, help="timed C3 decodes per engine and round")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_engines.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    tts = bench.build_product(dev)
    wav_h, phone_h, forced = bench.make_inputs(range(bench.B_PER_GPU))
    wav, phone, forced = wav_h.to(dev), phone_h.to(dev), forced.to(dev)
    g = torch.Generator().manual_seed(bench.SEED0 + 3)
    tc = torch.relu(torch.randn(16, 512, 512, generator=g)).to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    step = lambda: bench.gpu_step(tts, wav, phone, forced)
    decode = lambda: tts.plm.infer(tc)
    card_before = card()

    res = {name: {"step_ms": [], "decode_ms": []} for name, _, _ in ENGINES}
    for r in range(args.rounds):
        for name, engine, _ in ENGINES:
            with pack.engine_scope(engine):
                for _ in range(4 if graphs.enabled() else 1):      # plans for this engine, graph capture, first replays
                    step()
                    decode()
                ms, _ = timed(step, args.steps, flush)
                res[name]["step_ms"].append(round(ms, 2))
                ms, _ = timed(decode, args.decodes)
                res[name]["decode_ms"].append(round(ms, 1))
            print(f"[bench_engines] round {r} {name}: step {res[name]['step_ms'][-1]} ms, decode {res[name]['decode_ms'][-1]} ms",
                  file=sys.stderr, flush=True)
    card_after = card()

    outs = {}
    pk, pk_src = bench.peaks()
    peak = float(pk.get("bf16_tflops_sustained", pk.get("bf16_tflops")))
    for name, engine, mpp in ENGINES:
        with pack.engine_scope(engine):
            outs[name] = (bench.gpu_step(tts, wav, phone, forced, intermediates=True), decode())
            torch.cuda.synchronize()
            ps = profile(lambda: bench.gpu_step(tts, wav, phone, forced, overlap=False))
            pd = profile(decode)
        r = res[name]
        for key, p in (("step", ps), ("decode", pd)):
            ach = p["tc_tflop"] / (p["tc_ms"] / 1e3) if p["tc_ms"] > 0 else 0.0
            r[f"tap_gemm_per_{key}"] = {"ms": round(p["tc_ms"], 1), "tflop": round(p["tc_tflop"], 2), "launches": p["tc_launches"],
                                        "achieved_tflops": round(ach, 1),
                                        "frac_of_scheme_ceiling": round(ach / (peak / mpp), 4)}
            r[f"ffma_per_{key}"] = {"ms": round(p["ffma_ms"], 1), "launches": p["ffma_launches"]}
        r.update(engine=name, mma_per_product=mpp, peak_tflops=peak, peak_source=f"{pk_src} dense fp16/bf16; the scheme's "
                 f"ceiling is peak / {mpp}", card_before=card_before, card_after=card_after,
                 workloads=f"C4 step: batch {bench.B_PER_GPU}, prompt re-vocode, L2 flush before each timed step; "
                           "C3 decode: MegaPLM.infer, 512 tokens, batch 16")
    base, base_ids = outs["f16x2"]
    for name, _, _ in ENGINES:
        o, ids = outs[name]
        res[name]["vs_f16x2"] = {
            "wav_max_abs_diff": float((o["wav"] - base["wav"]).abs().max()),
            "mel_l1": float((o["mel"] - base["mel"]).abs().mean()),
            "c4_p_codes_agreement": float((o["p_codes"] == base["p_codes"]).double().mean()),
            "c4_dt_agreement": float((o["dt"] == base["dt"]).double().mean()),
            "c3_ids_agreement": float((ids == base_ids).double().mean()),
            "all_finite": bool(torch.isfinite(o["wav"]).all() and torch.isfinite(o["mel"]).all()),
        }
        print(json.dumps(res[name]), flush=True)


if __name__ == "__main__":
    main()
