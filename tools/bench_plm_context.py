"""Cost of in-context prompting of the prosody LM, at T = 64 target steps, B = 1, 16, 64 and P = 0, 32, 64, 128 context rows:

- the non-causal context decode (MegaPLM.infer(..., context=...)) against the decode it must equal, the existing range
  driver over a materialised cat(ctx_tc, tc) with the context codes prefilled, run over [P, P+T) (MegaPLM.begin_decode on
  the concatenation + decode_until); both replay as CUDA graphs; the modelled encoder-row ratio against P = 0,
  (P*T + T^2/2) / (T^2/2), is printed beside them;
- the causal context decode (MegaPLM.infer_causal(..., context=...)) against infer_causal without a context, with its
  prefill estimated as the context decode at T = 1 minus the plain causal decode at T = 1;
- a C4 synthesize (bench.py's workload, batch 64) with one shared 64-row context against the same call without it.

Arms alternate within each round.  GPU only; prints JSON lines, the card's name, power limit and maximum SM clock first.

    python tools/bench_plm_context.py [--rounds 3] [--skip-c4]
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

T = 64


def context(Bc, P, seed):
    from megatts2_b200.models.megatts2 import PLMContext
    g = torch.Generator().manual_seed(seed)
    return PLMContext(F.relu(torch.randn(Bc, P, 512, generator=g)).to(DEV),
                      torch.randint(0, 1024, (Bc, P), generator=g).to(DEV))


def cat_range(plm, cat, codes, P):
    """The range driver over the materialised concatenation, steps [P, P+T), context codes prefilled."""
    dec = plm.begin_decode(cat)
    dec.state[:, 1:P + 1] = codes
    dec.t = P
    return plm.decode_until(dec, P + T)


def rounds_for(plm, B, P, rounds):
    g = torch.Generator().manual_seed(100 + B)
    tc = F.relu(torch.randn(B, T, 512, generator=g)).to(DEV)
    arms = {"plain_infer": lambda: plm.infer(tc), "plain_causal": lambda: plm.infer_causal(tc),
            "plain_causal_T1": lambda: plm.infer_causal(tc[:, :1])}
    if P:
        ctx = context(1, P, 7 + P)
        cat = torch.cat([ctx.tc8.expand(B, -1, -1), tc], 1).contiguous()
        codes = ctx.codes.expand(B, -1)
        arms.update(ctx_infer=lambda: plm.infer(tc, context=ctx), cat_range=lambda: cat_range(plm, cat, codes, P),
                    ctx_causal=lambda: plm.infer_causal(tc, context=ctx),
                    ctx_causal_T1=lambda: plm.infer_causal(tc[:, :1], context=ctx))
        assert torch.equal(arms["ctx_infer"](), arms["cat_range"]())           # the two non-causal arms decode the same
    for fn in arms.values():               # eager run + CUDA-graph capture of every arm before anything is timed
        for _ in range(3):
            fn()
    times = {n: [] for n in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            times[name].append(timed_ms(fn))
    out = {"B": B, "P": P, "T": T, "model_rows_ratio": round((P * T + T * T / 2) / (T * T / 2), 2)}
    out.update({n + "_ms": [round(v, 3) for v in t] for n, t in times.items()})
    if P:
        out["ctx_vs_cat_range_pct"] = [round(100 * (a / b - 1), 2) for a, b in zip(times["ctx_infer"], times["cat_range"])]
        out["ctx_vs_plain_infer_x"] = [round(a / b, 2) for a, b in zip(times["ctx_infer"], times["plain_infer"])]
        out["causal_prefill_ms"] = [round(a - b, 3) for a, b in zip(times["ctx_causal_T1"], times["plain_causal_T1"])]
        out["causal_steps_ms"] = [round(c - (a - b), 3) for a, b, c in zip(times["ctx_causal_T1"],
                                                                           times["plain_causal_T1"], times["ctx_causal"])]
    print(json.dumps(out), flush=True)


def c4_rounds(rounds):
    import bench
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    dev = torch.device(DEV)
    tts = bench.build_product(dev)
    wav, phone, forced = bench.make_inputs(range(bench.B_PER_GPU))
    wav, phone, forced = wav.to(dev), phone.to(dev), forced.to(dev)
    ctx = context(1, 64, 5)

    def step(with_ctx):
        mel = extract_mel_spec(wav, frames_major=True)
        return tts.synthesize(phone, mel, forced_durations=forced, prompt_mels=mel,
                              plm_context=ctx if with_ctx else None)

    for c in (False, True):
        for _ in range(3):
            step(c)
    times = {"plain": [], "context64": []}
    for _ in range(rounds):
        for name, c in (("plain", False), ("context64", True)):
            times[name].append(timed_ms(lambda: step(c)))
    print(json.dumps({"c4_B": bench.B_PER_GPU, **{n + "_ms": [round(v, 1) for v in t] for n, t in times.items()},
                      "context_vs_plain_pct": [round(100 * (a / b - 1), 2) for a, b in zip(times["context64"],
                                                                                           times["plain"])]}), flush=True)


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
    print(json.dumps({"setup_s": round(time.time() - t0, 1)}), flush=True)
    for B in (1, 16, 64):
        for P in (0, 32, 64, 128):
            rounds_for(plm, B, P, args.rounds)
    del plm
    torch.cuda.empty_cache()
    if not args.skip_c4:
        c4_rounds(args.rounds)


if __name__ == "__main__":
    main()
