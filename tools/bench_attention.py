"""A/B of the two attention kernels (diagnostics, GPU only) at the PLM / ADM head shapes, sequence lengths 32 .. 512, in
one process: under the bf16x3 engine every call runs the fp32 FFMA kernel (ops.cu); under f16x2 sequences of 65 rows or
more run the wgmma kernel (attn_tc.cu), shorter ones stay on the fp32 kernel unless MEGATTS2_ATTN_PAIR_MIN routes them."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megatts2_b200 import ops, pack  # noqa: E402

ENGINES = (("bf16x3", pack.ENGINE_BF16X3), ("f16x2", pack.ENGINE_F16X2))


def time_ms(f, reps=20):
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    pair_min = os.environ.get("MEGATTS2_ATTN_PAIR_MIN", "off")
    for (B, H, dh) in ((64, 16, 64), (64, 8, 96), (16, 16, 64)):
        for S in [int(x) for x in os.environ.get("BENCH_S", "32,64,128,256,512").split(",")]:
            if B * S > 64 * 256 and B == 64:
                continue
            qkv = torch.randn(B, S, 3 * H * dh, device="cuda")
            D = H * dh
            f = lambda: ops.attention(qkv[..., :D], qkv[..., D:2 * D], qkv[..., 2 * D:], H)
            fl = 4.0 * B * H * S * S * dh
            for name, engine in ENGINES:
                with pack.engine_scope(engine):
                    ms = time_ms(f)
                print(f"{name:6s} PAIR_MIN={pair_min} B{B} H{H} dh{dh} S{S:4d}: {ms * 1e3:8.1f} us  {fl / ms / 1e9:7.2f} TFLOP/s", flush=True)


if __name__ == "__main__":
    main()
