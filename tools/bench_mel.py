#!/usr/bin/env python
"""Config C2: STFT + mel-filterbank kernel on 10k synthetic 16 kHz 3-s clips, one GPU.
Prints one JSON line: clips/s, achieved algorithmic GB/s (252,160 B per clip: 192,000 in + 60,160 out)
and the fraction of the measured HBM peak."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1235)
    wav = torch.rand(n, 48000, device=dev, generator=g) * 2 - 1        # 1.92 GB >> 126 MB L2
    for _ in range(3):
        out = extract_mel_spec(wav)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    e0.record()
    for _ in range(reps):
        out = extract_mel_spec(wav)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    bytes_alg = n * (48000 * 4 + 80 * 188 * 4)
    gbs = bytes_alg / (ms / 1e3) / 1e9
    pk = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
        os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0      # H100 SXM data sheet
    frames = n * 188
    print(json.dumps({"config": "C2 mel front end", "clips": n, "ms": round(ms, 4), "clips_per_s": round(n / (ms / 1e3)),
                      "frames_per_s": round(frames / (ms / 1e3)), "achieved_gbs": round(gbs, 1), "peak_gbs": pk,
                      "frac_hbm": round(gbs / pk, 4), "out_shape": list(out.shape)}))


if __name__ == "__main__":
    main()
