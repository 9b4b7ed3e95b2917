#!/usr/bin/env python
"""Streamed synthesis latency: ``Megatts.synthesize_stream`` against ``synthesize`` on bench.py's utterances (U: 64 phones
x 8 frames = 512 mel frames, 64 PLM steps; no prompt re-vocode; default engine).

For B in {1, 64} and chunk_frames in {32, 64, 128}: the time to the first synthesized chunk and to the last one (host
clock from the call to the synchronise after that chunk is yielded), every chunk's time, and the ``synthesize`` time (host
clock to its synchronise), in three alternated rounds after two untimed set-up rounds (plans, graph captures).  Each
stream's output is compared with ``synthesize``'s.  The halo share is modelled: the decoder + vocoder time of one
full-length run (CUDA events) times the extra window frames the schedule recomputes over L.  Results: one JSON line per
(B, chunk_frames) and a Markdown table, also written to --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def time_synth(tts, phone, mel, forced):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = tts.synthesize(phone, mel, forced_durations=forced, return_intermediates=True)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def time_stream(tts, phone, mel, forced, cf):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    marks, chunks = [], []
    for c in tts.synthesize_stream(phone, mel, forced_durations=forced, chunk_frames=cf):
        torch.cuda.synchronize()
        marks.append(time.perf_counter() - t0)
        chunks.append(c)
    return marks, chunks


def halo_frames(tts, L, cf):
    from megatts2_b200 import stream as SCH
    gen, voc = tts.generator, tts.hifi_gan.generator
    plan = SCH.schedule(L, cf, gen.decoder.receptive_field(), voc.receptive_field(), voc.cfg["inference_padding"])
    dec = sum(c.dec[1] - c.dec[0] for c in plan if c.dec is not None)
    vo = sum(c.voc[1] - c.voc[0] for c in plan)
    return dec, vo


def dec_voc_ms(tts, out):
    """CUDA-event time of the full-length mel decoder and vocoder on synthesize's own intermediates (median of 5)."""
    ts = []
    for _ in range(6):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        mel = tts.generator.decode_mel_cl(out["tc_latent_expand"], out["p_codes"])
        e[1].record()
        tts.hifi_gan.decode_batch_cl(mel)
        e[2].record()
        torch.cuda.synchronize()
        ts.append((e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])))
    return statistics.median(t[0] for t in ts[1:]), statistics.median(t[1] for t in ts[1:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,64")
    ap.add_argument("--chunks", default="32,64,128")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines and the table here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device: bench_stream measures the CUDA path only"}))
        sys.exit(1)
    import ctypes as C
    from megatts2_b200 import _lib as L
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card()
    tts = bench.build_product(dev)
    T = -(-bench.TP * bench.DUR // 8)
    lines, rows = [], []
    for B in [int(x) for x in args.batches.split(",")]:
        wav, phone, forced = bench.make_inputs(range(B), pin=False)
        wav, phone, forced = wav.to(dev), phone.to(dev), forced.to(dev)
        mel = extract_mel_spec(wav, frames_major=True)
        ws_mib = L.lib().mtts_plm_infer_workspace_bytes(C.byref(tts.plm._plan_get(dev, T).struct), B, T) / 2 ** 20
        for cf in [int(x) for x in args.chunks.split(",")]:
            # the stream's range graphs (8 per model) hold one chunk_frames value at a time, so the set-up (plans,
            # workspaces, captures) and the alternated rounds pair synthesize with one chunk_frames value
            for _ in range(2):
                time_synth(tts, phone, mel, forced)
                time_stream(tts, phone, mel, forced, cf)
            synth, runs = [], []
            for _ in range(args.rounds):
                t, ref = time_synth(tts, phone, mel, forced)
                synth.append(t)
                runs.append(time_stream(tts, phone, mel, forced, cf))
            dec_ms, voc_ms = dec_voc_ms(tts, ref)
            L_ = max(ref["totals"])
            marks, chunks = [m for m, _ in runs], runs[-1][1]
            w = torch.cat([c["wav"] for c in chunks], -1)
            err = (w - ref["wav"]).abs().max().item()
            codes_equal = bool(torch.equal(chunks[-1]["p_codes"], ref["p_codes"]))
            dec_f, voc_f = halo_frames(tts, L_, cf)
            halo_ms = dec_ms * (dec_f - L_) / L_ + voc_ms * (voc_f - L_) / L_
            ms = lambda x: round(x * 1e3, 2)
            res = dict(card=info, B=B, chunk_frames=cf, L=L_, T=T, n_chunks=len(chunks),
                       first_chunk_ms=ms(statistics.median(m[0] for m in marks)),
                       last_chunk_ms=ms(statistics.median(m[-1] for m in marks)),
                       synthesize_ms=ms(statistics.median(synth)),
                       per_chunk_ms=[ms(statistics.median(m[i] - (m[i - 1] if i else 0) for m in marks))
                                     for i in range(len(marks[0]))],
                       rounds_first_ms=[ms(m[0]) for m in marks], rounds_last_ms=[ms(m[-1]) for m in marks],
                       rounds_synthesize_ms=[ms(x) for x in synth],
                       decoder_window_frames=dec_f, vocoder_window_frames=voc_f,
                       full_decoder_ms=round(dec_ms, 2), full_vocoder_ms=round(voc_ms, 2),
                       halo_ms_modelled=round(halo_ms, 2), plm_workspace_mib_per_graph=round(ws_mib, 1),
                       max_abs_vs_synthesize=err, codes_equal=codes_equal, bit_identical=bool(torch.equal(w, ref["wav"])))
            lines.append(json.dumps(res))
            print(lines[-1], flush=True)
            rows.append(f"| {B} | {cf} | {len(chunks)} | {res['first_chunk_ms']} | {res['last_chunk_ms']} | "
                        f"{res['synthesize_ms']} | {res['halo_ms_modelled']} | {err:.1e} | {'yes' if codes_equal else 'NO'} |")
    table = [f"card: {info}", "",
             "| B | chunk_frames | chunks | first chunk ms | last chunk ms | synthesize ms | halo ms (modelled) | "
             "max abs vs synthesize | codes equal |",
             "|---|---|---|---|---|---|---|---|---|"] + rows
    print("\n".join(table))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines + [""] + table) + "\n")


if __name__ == "__main__":
    main()
