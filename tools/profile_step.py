#!/usr/bin/env python
"""One bench step between cudaProfilerStart/Stop, for `ncu --profile-from-start off`.

    ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv \
        --log-file launches.csv python tools/profile_step.py [--batch 64]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--stage", default="all", choices=["all", "mel", "hifigan", "plm"])
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    tts = bench.build_product(dev)
    wav, phone, forced = bench.make_inputs(range(a.batch))
    wav, phone, forced = wav.to(dev), phone.to(dev), forced.to(dev)
    from megatts2_b200 import ops
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    bench.gpu_step(tts, wav, phone, forced)          # warm-up: plans, workspace, attributes
    torch.cuda.synchronize()
    rt = torch.cuda.cudart()
    if a.stage == "all":
        rt.cudaProfilerStart()
        bench.gpu_step(tts, wav, phone, forced, overlap=False)
        torch.cuda.synchronize()
        rt.cudaProfilerStop()
        return
    mel = extract_mel_spec(wav, frames_major=True)
    if a.stage == "mel":
        torch.cuda.synchronize()
        rt.cudaProfilerStart()
        extract_mel_spec(wav, frames_major=True)
        torch.cuda.synchronize()
        rt.cudaProfilerStop()
        return
    tc = tts.generator.mrte.tc_latent(phone, mel)
    exp = tts.lr(tc, forced)
    tc8 = ops.maxpool_time(exp, 8)
    if a.stage == "plm":
        torch.cuda.synchronize()
        rt.cudaProfilerStart()
        tts.plm.infer(tc8)
        torch.cuda.synchronize()
        rt.cudaProfilerStop()
        return
    codes = tts.plm.infer(tc8)
    melo = tts.generator.decode_mel_cl(exp, codes)
    torch.cuda.synchronize()
    rt.cudaProfilerStart()
    tts.hifi_gan.decode_batch_cl(melo)
    torch.cuda.synchronize()
    rt.cudaProfilerStop()


if __name__ == "__main__":
    main()
