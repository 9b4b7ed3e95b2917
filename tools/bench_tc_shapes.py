"""Per-shape throughput of the tensor-core tap-GEMM (diagnostics, GPU only).

For each shape runs the op `reps` times inside the library's event trace and reports the main kernel's
time per launch (the activation split is traced separately) and its rate in fp32-equivalent TFLOP/s
(2*M*N*K*k; the tensor pipe executes 6 | 3 | 1 16-bit MMAs per product under bf16x3 | f16x2 | f16, so the dense
16-bit rate is that multiple of it), and the operand bytes the launch plan moves from L2 into the SMs (modelled from the
plan, not measured) with their rate.
"""
import ctypes as C
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megatts2_b200 import _lib as L, ops, pack  # noqa: E402

DEV = "cuda:0"
SHAPES = [
    # PLM / ADM dense layers (k = 1): rows = batch x sequence
    dict(name="plm qkv  M5888 K1024 N3072", B=1, T=5888, Cin=1024, Cout=3072, k=1),
    dict(name="plm ff1  M5888 K1024 N4096", B=1, T=5888, Cin=1024, Cout=4096, k=1),
    dict(name="plm ff2  M5888 K4096 N1024", B=1, T=5888, Cin=4096, Cout=1024, k=1),
    dict(name="plm out  M5888 K1024 N1024", B=1, T=5888, Cin=1024, Cout=1024, k=1),
    # HiFi-GAN ResBlock convs
    dict(name="hifi s1  C256 k7  T4176 B64", B=64, T=4176, Cin=256, Cout=256, k=7, dil=3),
    dict(name="hifi s2  C128 k7  T8352 B64", B=64, T=8352, Cin=128, Cout=128, k=7, dil=3),
    dict(name="hifi s3  C64  k7  T33408 B64", B=64, T=33408, Cin=64, Cout=64, k=7, dil=3),
    dict(name="hifi s4  C32  k7  T66816 B64", B=64, T=66816, Cin=32, Cout=32, k=7, dil=3),
    # AR-loop shapes at smaller steps (rows = 64 x t)
    dict(name="plm ff1  M2048 K1024 N4096", B=1, T=2048, Cin=1024, Cout=4096, k=1),
    dict(name="plm ff2  M2048 K4096 N1024", B=1, T=2048, Cin=4096, Cout=1024, k=1),
    dict(name="plm qkv  M1024 K1024 N3072", B=1, T=1024, Cin=1024, Cout=3072, k=1),
    dict(name="adm qkv  M4096 K768  N2304", B=1, T=4096, Cin=768, Cout=2304, k=1),
    dict(name="adm ff1  M4096 K768  N1024", B=1, T=4096, Cin=768, Cout=1024, k=1),
]


def operand_bytes(s, fmt, sms):
    """L2 -> SM operand bytes of one launch, modelled from the plan (mtts_tc_plan_query_ex): every CTA work item loads,
    per K-slab, its activation tile and the weight tile (or, in a 2-CTA cluster, half of it; a dummy item included) of
    each operand plane; the halo form loads the activation tile with its halo once per item.  Returns (bytes, plan)."""
    k, dil = s["k"], s.get("dil", 1)
    out = (C.c_int32 * 7)()
    L.check(L.lib().mtts_tc_plan_query_ex(sms, s["B"], s["T"], s["Cin"], s["Cout"], k, dil, fmt, 0, 0,
                                          ops.launch_policy_now()[1], out))
    bn, splits, halo, swb, cl = out[0], out[1], out[3], out[4], out[5]
    npl = 3 - fmt
    rows = 128 if (halo or bn != 128) else 64
    rt = s["B"] * -(-s["T"] // rows)
    nt = -(-s["Cout"] // bn)
    nk = k * -(-s["Cin"] // (swb // 2))
    if halo:
        return rt * nt * npl * ((128 + dil * (k - 1)) * swb + nk * bn * swb), out
    cta_items = (2 * -(-rt // 2) if cl == 2 else rt) * nt
    return cta_items * nk * npl * (rows * swb + bn * swb // cl), out


def trace_ms(fn, reps):
    lib = L.lib()
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    lib.mtts_trace_begin(ops._stream())
    for _ in range(reps):
        fn()
    buf = C.create_string_buffer(16384)
    lib.mtts_trace_end(buf, 16384)
    for line in buf.value.decode().splitlines():
        f = line.split()
        if f and f[0] == "conv_tc_launch":
            return float(f[2]) / int(f[1])
    return float("nan")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--shapes", type=str, default="", help="comma-separated shape indices (default: all)")
    ap.add_argument("--fmt", type=str, default="f16x2", choices=["f16x2", "bf16x3", "f16"])
    args = ap.parse_args()
    reps = args.reps
    shapes = [SHAPES[int(i)] for i in args.shapes.split(",")] if args.shapes else SHAPES
    g = torch.Generator().manual_seed(0)
    for s in shapes:
        k, dil = s["k"], s.get("dil", 1)
        pad = dil * (k - 1) // 2
        x = torch.randn(s["B"], s["T"], s["Cin"], generator=g).to(DEV)
        w = torch.randn(s["Cout"], s["Cin"], k, generator=g) / math.sqrt(s["Cin"] * k)
        b = torch.randn(s["Cout"], generator=g).to(DEV)
        fmt = {"f16x2": pack.FMT_F16X2, "bf16x3": pack.FMT_BF16X3, "f16": pack.FMT_F16}[args.fmt]
        nm = {pack.FMT_F16X2: 3, pack.FMT_BF16X3: 6, pack.FMT_F16: 1}[fmt]
        wp, wt = pack.pack_conv(w.to(DEV)), pack.pack_conv_tc_planes(w.to(DEV), fmt)
        out = torch.empty(s["B"], s["T"], s["Cout"], device=DEV)
        flops = 2.0 * s["B"] * s["T"] * s["Cin"] * s["Cout"] * k
        ms = trace_ms(lambda: ops.conv1d(x, wp, b, out=out, w_tc=wt, k=k, dil=dil, pad=pad, pad_mode=1 if k > 1 else 0), reps)
        nbytes, plan = operand_bytes(s, fmt, ops.sm_count(torch.device(DEV)))
        print(f"{s['name']:30s} {ms:8.3f} ms  {flops / ms / 1e9:7.1f} TFLOP/s per product "
              f"({nm * flops / ms / 1e9:7.0f} dense 16-bit, {args.fmt})  L2->SM {nbytes / 1e9:6.2f} GB "
              f"{nbytes / ms / 1e9:5.2f} TB/s  (BN {plan[0]}, cluster {plan[5]})", flush=True)
        del x, out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
