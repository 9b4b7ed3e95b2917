"""Cost of speech editing, on bench.py's utterance (64 phones of 8 frames: 512 frames, T = 64 PLM steps).

1. MegaPLM.infer(pinned=) against infer at B = 1, 16, 64: spans of 1, 3 and 8 phones at the start, the middle and the
   end, every other step pinned to infer's own codes, so the pinned decode runs the span's steps only.
2. The pinned ADM decode alone (every phone runs; an ADM range driver is not built), so the cost an edit keeps is visible.
3. Megatts.edit (a replacement by as many new phones, span_frames = the replaced frames) against synthesize with the
   original's forced durations, at the same sizes.

Arms alternate within each round.  GPU only; prints JSON lines, the card's name, power limit and maximum SM clock first.

    python tools/bench_speech_edit.py [--rounds 3] [--skip-edit]
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

T, TP, DUR = 64, 64, 8
SPANS = (1, 3, 8)


def starts(n):
    return {"start": 0, "middle": (TP - n) // 2, "end": TP - n}


def rounds_of(arms, rounds):
    for fn in arms.values():               # eager run + CUDA-graph capture of every arm before anything is timed
        for _ in range(3):
            fn()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed_ms(fn))
    return times


def plm_rounds(plm, B, rounds):
    g = torch.Generator().manual_seed(11 + B)
    tc = F.relu(torch.randn(B, T, 512, generator=g)).to(DEV)
    codes = plm.infer(tc).cpu().to(torch.int32)
    for n in SPANS:
        for where, a in starts(n).items():
            pins = codes.clone()
            pins[:, a:a + n] = -1
            t = rounds_of({"infer": lambda: plm.infer(tc), "pinned": lambda: plm.infer(tc, pinned=pins)}, rounds)
            print(json.dumps({"plm_B": B, "T": T, "free_steps": n, "where": where,
                              **{k + "_ms": [round(v, 3) for v in x] for k, x in t.items()},
                              "pinned_vs_infer_pct": [round(100 * (p / i - 1), 2) for p, i in zip(t["pinned"],
                                                                                                 t["infer"])]}),
                  flush=True)
        plm._graphs("pinned").clear()      # a captured graph pins its workspace


def adm_rounds(adm, B, rounds):
    g = torch.Generator().manual_seed(21 + B)
    tc = F.relu(torch.randn(B, TP, 512, generator=g)).to(DEV)
    pins = torch.full((B, TP), DUR, dtype=torch.int32)
    pins[:, 30:33] = -1
    t = rounds_of({"adm": lambda: adm.infer(tc), "adm_pinned": lambda: adm.infer(tc, pinned=pins)}, rounds)
    print(json.dumps({"adm_B": B, "Tp": TP, **{k + "_ms": [round(v, 3) for v in x] for k, x in t.items()}}), flush=True)


def edit_rounds(tts, B, rounds):
    import bench
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    wav, phone, forced = bench.make_inputs(range(B))
    wav, phone, forced = wav.to(DEV), phone.to(DEV), forced.to(DEV)
    mel = extract_mel_spec(wav, frames_major=True)
    orig = tts.synthesize(phone, mel, forced_durations=forced, return_intermediates=True)
    for n in SPANS:
        for where, a in starts(n).items():
            edited = phone.clone()
            edited[:, a:a + n] = (edited[:, a:a + n] + 1) % 320
            span = torch.tensor([[a, a + n]] * B)
            sf = [n * DUR] * B
            t = rounds_of({"synthesize": lambda: tts.synthesize(phone, mel, forced_durations=forced),
                           "edit": lambda: tts.edit(edited, mel, phone, forced, orig["p_codes"], span, span_frames=sf)},
                          rounds)
            print(json.dumps({"edit_B": B, "span_phones": n, "where": where,
                              **{k + "_ms": [round(v, 1) for v in x] for k, x in t.items()},
                              "edit_vs_synthesize_pct": [round(100 * (e / s - 1), 2) for e, s in zip(t["edit"],
                                                                                                    t["synthesize"])]}),
                  flush=True)
        tts.plm._graphs("pinned").clear()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-edit", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        sys.exit(1)
    print(json.dumps({"card": card()}), flush=True)
    t0 = time.time()
    plm = helpers.build_plm(weights.plm_state_dict(), DEV)
    adm = helpers.build_adm(weights.adm_state_dict(), DEV)
    print(json.dumps({"setup_s": round(time.time() - t0, 1)}), flush=True)
    for B in (1, 16, 64):
        plm_rounds(plm, B, args.rounds)
        adm_rounds(adm, B, args.rounds)
    del plm, adm
    torch.cuda.empty_cache()
    if not args.skip_edit:
        import bench
        tts = bench.build_product(torch.device(DEV))
        for B in (1, 16, 64):
            edit_rounds(tts, B, args.rounds)


if __name__ == "__main__":
    main()
