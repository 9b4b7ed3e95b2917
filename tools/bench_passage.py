"""Cost of long-form synthesis on bench.py's C4 utterance (64 phones, durations forced to 8: 512 frames and T = 64 PLM
steps per sentence, an 8-s prompt of 500 frames), for passages of S in {4, 10} sentences at B in {1, 16}, plus one
ragged-duration case (durations 1..15).  Arms, alternating within each round:

  passage      synthesize_passage at the default window (128 rows)
  passage_cr0  synthesize_passage with context_rows=0 (independent sentences, one vocoder pass)
  separate     S synthesize calls, one per sentence (graphed AR decodes, as a caller gets them)
  oneshot      one synthesize over the S x 64 concatenated phones (the quadratic PLM decode)
  stream       synthesize_passage_stream: time to the first and to the last chunk

and, per B, one sentence with the AR decodes eager (graphs.disabled(), as a passage runs them) against graphed.  The
outputs are compared across arms: the passage at context_rows=0 against the separate calls (codes), the stream against
the whole call (samples).  GPU only; prints JSON lines, the card's name, power limit and maximum SM clock first.

    python tools/bench_passage.py [--rounds 2] [--S 4,10] [--B 1,16] [--skip-oneshot]
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
from megatts2_b200 import graphs  # noqa: E402
from oracle import weights  # noqa: E402  (seeded weight specs only; nothing of the oracle is timed here)

TP, TM, DUR = 64, 500, 8


def inputs(S, B, ragged, seed=7):
    g = torch.Generator().manual_seed(seed + S + B)
    sents = [torch.randint(0, 320, (B, TP), generator=g).to(DEV) for _ in range(S)]
    forced = [(torch.randint(1, 16, (B, TP), generator=g, dtype=torch.int32) if ragged else
               torch.full((B, TP), DUR, dtype=torch.int32)).to(DEV) for _ in range(S)]
    mel = (torch.randn(B, TM, 80, generator=g) * 2 - 4).to(DEV)
    return sents, forced, mel


def stream_ms(tts, sents, mel, forced):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, wavs = None, []
    for c in tts.synthesize_passage_stream(sents, mel, forced_durations=forced, pause_frames=16):
        torch.cuda.synchronize()
        if first is None:
            first = 1e3 * (time.perf_counter() - t0)
        wavs.append(c)
    return first, 1e3 * (time.perf_counter() - t0), wavs


def case(tts, S, B, ragged, rounds, skip_oneshot):
    sents, forced, mel = inputs(S, B, ragged)
    cat_ph, cat_fd = torch.cat(sents, 1), torch.cat(forced, 1)
    arms = {
        "passage": lambda: tts.synthesize_passage(sents, mel, forced_durations=forced, pause_frames=16),
        "passage_cr0": lambda: tts.synthesize_passage(sents, mel, forced_durations=forced, pause_frames=16,
                                                      context_rows=0),
        "separate": lambda: [tts.synthesize(p, mel, forced_durations=f) for p, f in zip(sents, forced)],
    }
    if not skip_oneshot:
        arms["oneshot"] = lambda: tts.synthesize(cat_ph, mel, forced_durations=cat_fd)
    for fn in arms.values():          # warm-up: plans, graphs of the separate calls, allocator
        fn()
        fn()
    times = {n: [] for n in arms}
    first, last = [], []
    for _ in range(rounds):
        for name, fn in arms.items():
            times[name].append(timed_ms(fn))
        f, la, _ = stream_ms(tts, sents, mel, forced)
        first.append(f)
        last.append(la)
    # outputs compared across arms
    whole = tts.synthesize_passage(sents, mel, forced_durations=forced, pause_frames=16, return_intermediates=True)
    cr0 = tts.synthesize_passage(sents, mel, forced_durations=forced, pause_frames=16, context_rows=0,
                                 return_intermediates=True)
    sep = [tts.synthesize(p, mel, forced_durations=f, return_intermediates=True) for p, f in zip(sents, forced)]
    codes_equal = all(torch.equal(a["p_codes"], b["p_codes"]) for a, b in zip(cr0["sentences"], sep))
    _, _, chunks = stream_ms(tts, sents, mel, forced)
    err = 0.0
    for b in range(B):
        row = torch.cat([c["wav"][b, 0, :c["valid"][b]] for c in chunks])
        err = max(err, (row - whole["wav"][b, 0, :row.numel()]).abs().max().item())
    print(json.dumps({"S": S, "B": B, "ragged": ragged, **{n + "_ms": [round(v, 1) for v in t] for n, t in times.items()},
                      "stream_first_ms": [round(v, 1) for v in first], "stream_last_ms": [round(v, 1) for v in last],
                      "context_rows_used": whole["context_rows_used"].tolist(),
                      "cr0_codes_equal_separate": codes_equal, "stream_vs_whole_max_abs": err}), flush=True)


def eager_vs_graphed(tts, B, rounds):
    sents, forced, mel = inputs(1, B, False)
    graphed = lambda: tts.synthesize(sents[0], mel, forced_durations=forced[0])  # noqa: E731

    def eager():
        with graphs.disabled():
            tts.synthesize(sents[0], mel, forced_durations=forced[0])
    for fn in (graphed, eager):
        fn()
        fn()
    t = {"graphed": [], "eager": []}
    for _ in range(rounds):
        t["graphed"].append(timed_ms(graphed))
        t["eager"].append(timed_ms(eager))
    print(json.dumps({"one_sentence_B": B, **{k + "_ms": [round(v, 1) for v in x] for k, x in t.items()}}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--S", default="4,10")
    ap.add_argument("--B", default="1,16")
    ap.add_argument("--skip-oneshot", action="store_true")
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    tts = helpers.build_megatts(weights.g_state_dict(), weights.plm_state_dict(), weights.adm_state_dict(),
                                weights.hifigan_state_dict(), DEV)
    Bs, Ss = [int(x) for x in args.B.split(",")], [int(x) for x in args.S.split(",")]
    for B in Bs:
        eager_vs_graphed(tts, B, args.rounds)
        for S in Ss:
            case(tts, S, B, False, args.rounds, args.skip_oneshot)
    case(tts, Ss[0], Bs[0], True, args.rounds, args.skip_oneshot)


if __name__ == "__main__":
    main()
