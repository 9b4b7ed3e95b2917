"""Every launch plan of the exact-fp32 FFMA tap-GEMM (csrc/tapconv.cu) against fp64.

``ffma_plan()`` picks what conv1d_ffma() launches for a call: the tiled or per-thread Cout = 1 kernel, the 64x64 tile with
K split over blockIdx.z plus splitk_reduce_kernel, or one of the tiles 128x32, 128x64, 128x128, 64x64; and the 16-byte
load / store paths vec_a (x), vec_b (w) and vec_y (y and res).  The split depends on the SM budget of the calling thread
(``ops.launch_policy``), so one table of cases runs at budgets 1, 3, 16, 100 and the full device; every run logs the plan
``mtts_ffma_plan_query`` reports for it and its error as a fraction of the bar.  Each case fills mtts_conv_params itself:
that is the only way in with split-K room (tc_scratch without w_tc), strided views, 4-byte offsets and in-place residuals.

Reference: fp64 over the exact fp32 inputs.  The pre-activation is applied to x in fp32 on the host (ReLU is exact, leaky
is one correctly rounded product, as in the kernel); padding, the convolution and the epilogue run in fp64.  Rows outside
an item's input follow the rule include/megatts2_b200.h states for in_lens: zero / replicate / one reflection, and zero
where the reflection of a short input is still outside.

Bar, per output element.  The kernel computes each element as one fp32 FMA chain in a known order: tap j outer, channel c
ascending (for every tile and both Cout = 1 kernels: the K loop order does not depend on BM, BN, TM or TN).  A split makes
one chain per K range, each from 0.f, and the reduction adds the range sums in z order from 0.f.  Step i of a chain
rounds its running sum S_i once, with an error below U |S_i|; the errors are independent, so their sum stays below
LAMBDA * U * sqrt(sum_i S_i^2) (Hoeffding, as in test_gpu_resblock_oracle.py) with S_i the running sums in the kernel's
order, computed in fp64 from the exact products.  Steps with a zero product (padding, channels past Cin) are exact and not
counted.  For a split, the running sums of the reduction (z >= 1) join the same sum.  Then every rounding of the epilogue
adds U |value| (bias add, leaky's product, residual add, scale, accumulate), tanhf adds TANH_ULPS ulp (2 U |value| each);
ReLU, leaky (slope < 1) and tanh are 1-Lipschitz, so the chain's bound passes through them, and the scale multiplies it.
The CPU test ``test_bar_rejects_tf32`` checks the bar has teeth: the same chain over TF32-rounded x and w (what a
tensor-core TF32 engine multiplies) misses it by at least 4x in every case and plan.

Bit identity (GPU): runs of one case with equal plans are bit-identical across budgets, a repeat launch is bit-identical,
and - every unsplit kernel computing an element with the same chain - one batch item launched alone equals its rows of the
batched launch whenever neither launch is split, even where the two take different tiles or Cout = 1 kernels.

Every buffer is NaN outside the elements the kernel may read (x columns past Cin, x / res offsets, the split scratch), and
y holds seeded values everywhere, so a read outside the operands shows as NaN and a stray write as a changed element."""
import ctypes as C
import functools
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from megatts2_b200 import _lib as L

DEV = "cuda"
gpu = pytest.mark.gpu
BUDGETS = (1, 3, 16, 100, 0)          # SM budgets of the launching thread; 0 = the whole device
H100_SMS = 132                        # the full device in the host-only plan checks
NONE, RELU, LEAKY, TANH = L.ACT_NONE, L.ACT_RELU, L.ACT_LEAKY, L.ACT_TANH
ZERO, REFLECT, REPLICATE = L.PAD_ZERO, L.PAD_REFLECT, L.PAD_REPLICATE
FFMA_NONE, TILE, SPLITK, COUT1, COUT1_TILED = -1, 0, 1, 2, 3          # MTTS_FFMA_*
KERNEL_NAMES = {TILE: "tile", SPLITK: "splitk", COUT1: "cout1", COUT1_TILED: "cout1_tiled"}
BAD_ARG = -1


def f32(v):
    """the fp32 value the kernel is given for a host float"""
    return float(torch.tensor(v, dtype=torch.float32))


PRE_SLOPE, POST_SLOPE = f32(0.1), f32(0.2)
U = 2.0 ** -24                   # fp32 unit roundoff
LAMBDA = 6.0                     # independent rounding errors: P(|sum| > 6 sqrt(sum bound^2)) < 2 exp(-18) (Hoeffding)
TANH_ULPS = 2                    # tanhf's maximum error (CUDA C Programming Guide, single-precision functions)
TEETH = 4.0                      # a TF32 engine must miss the bar by at least this factor

# the dense layers of the AR decodes (causal_step, csrc/drivers.cu): (d_model, ff_dim); QKV is 3 d_model wide
PLM_D, PLM_F = 1024, 4096        # MegaPLM: d_model = vq_dim + tc_latent_dim (512 + 512), ff_dim = 4 d_model
ADM_D, ADM_F = 768, 1024         # MegaADM: d_model = emb_dim + tc_emb_dim (256 + 512), ff_dim = 4 emb_dim
DECODE_ROWS = (1, 5, 64, 65, 128, 200)


# ------------------------------------------------------------------------------------------ the case table
def _conv(B, T, Cin, Cout, k=1, **kw):
    return dict(B=B, T=T, Cin=Cin, Cout=Cout, k=k, **kw)


def _dense(M, K, N, **kw):
    return dict(B=1, T=M, Cin=K, Cout=N, k=1, **kw)


def _convt(B, T, Cin, Cout, s, **kw):
    """ConvTranspose1d(Cin, Cout, 2s, stride s, padding s/2) of the vocoder: a 2-tap conv with s * Cout columns over the
    leaky input, written at a negative output shift and clipped to the s T outputs"""
    return dict(B=B, T=T, Cin=Cin, Cout=Cout, s=s, k=2, pre=LEAKY, bias=True, **kw)


def _decode_scratch(M, D, F_):
    """the split-K room causal_take() gives every decode layer: 16 B wide floats + 4096 bytes"""
    return 16 * M * max(3 * D, F_) * 4 + 4096


# name -> case.  Keys: B, T (input rows), Cin, Cout, k, stride, dil, pad (default dil (k - 1) / 2), pad_mode; pre / post
# (activations), bias, res ("sep": own buffer, "inplace": res == y), acc (accumulate into y), scale (out_scale); ldx, xoff
# (x's channel stride and its offset in floats), ldy, yoff, ldr, roff; lens (in_lens); scratch (split-K room in bytes);
# s (the transposed-conv form).
CASES = {
    # ---- the shapes of the former parity table (ops.conv1d, bias on every one)
    "parity_m300_k1024_n4096": _conv(1, 300, 1024, 4096, bias=True),
    "parity_b4_t700_n1024_res": _conv(4, 700, 1024, 1024, bias=True, res="sep"),
    "parity_cin20_cout384_k5": _conv(2, 125, 20, 384, 5, bias=True),
    "parity_cin512_cout80_k5": _conv(2, 131, 512, 80, 5, bias=True),
    "parity_conv_post_b3": _conv(3, 257, 32, 1, 7, pad_mode=REFLECT, pre=LEAKY, post=TANH, bias=True),
    "parity_conv_post_t5000": _conv(2, 5000, 32, 1, 7, pad_mode=REFLECT, pre=LEAKY, post=TANH, bias=True),
    "parity_mrte_stride16": _conv(2, 500, 512, 512, 17, stride=16, pad=8, bias=True),
    "parity_c64_k11_dil5": _conv(2, 200, 64, 64, 11, dil=5, pad_mode=REFLECT, pre=LEAKY, bias=True, res="sep", acc=True,
                                 scale=1 / 3),
    "parity_c32_k3_dil3": _conv(2, 333, 32, 32, 3, dil=3, pad_mode=REFLECT, pre=LEAKY, bias=True),
    "parity_cin7_cout5_k3": _conv(1, 97, 7, 5, 3, bias=True),
    "parity_b5_t1_n768_res": _conv(5, 1, 768, 768, bias=True, res="sep"),
    "parity_b64_t1_k4096_n1024_res": _conv(64, 1, 4096, 1024, bias=True, res="sep"),
    "parity_m64_n4096_relu": _conv(1, 64, 1024, 4096, post=RELU, bias=True),
    "parity_b16_t2_k1000_n1000": _conv(16, 2, 1000, 1000, bias=True),
    "parity_conv_pre_k7": _conv(2, 64, 80, 512, 7, pad_mode=REFLECT, bias=True),
    "parity_cin16_cout24_replicate": _conv(2, 50, 16, 24, 5, pad_mode=REPLICATE, bias=True),
    # in_lens with zero padding over a channel slice (ldx 48, channels 8..31)
    "parity_in_lens_slice": _conv(3, 40, 24, 16, 5, ldx=48, xoff=8, lens=(40, 17, 29)),
    "parity_convt_s8": _convt(2, 37, 512, 256, 8),
    "parity_convt_s2": _convt(3, 301, 128, 64, 2),
    # ---- tile edges: Cout 32 / 33 and 64 / 65, 119 / 120 tiles of 128 x 128 (M tails on both sides)
    "cout32": _conv(2, 300, 48, 32, 3, bias=True, post=LEAKY),
    "cout33": _conv(2, 300, 48, 33, 3, bias=True, res="sep"),
    "cout64": _conv(2, 300, 48, 64, 3, pad_mode=REPLICATE, bias=True),
    "cout65": _conv(2, 300, 48, 65, 3, bias=True, acc=True),
    "tiles128_119": _conv(1, 15200, 16, 128, bias=True),
    "tiles128_120": _conv(1, 15300, 16, 128, bias=True, post=RELU),
    # ---- the Cout = 1 kernels: M 4095 / 4096, Cin 128 / 132, the tiled form's 48 KB of shared memory (dil 13: 48 992
    # bytes, dil 14: 49 856), stride 2, x not 16-byte aligned, k Cin above 8192, in_lens (a reflect halo of 3 rows)
    "cout1_m4095": _conv(1, 4095, 32, 1, 7, pad_mode=REFLECT, pre=LEAKY, post=TANH, bias=True),
    "cout1_m4096": _conv(1, 4096, 32, 1, 7, pad_mode=REFLECT, pre=LEAKY, post=TANH, bias=True),
    "cout1_cin128": _conv(1, 5000, 128, 1, 3, bias=True, res="sep"),
    "cout1_cin132": _conv(1, 5000, 132, 1, 3, pad_mode=REPLICATE, bias=True, acc=True, scale=0.5),
    "cout1_smem_dil13": _conv(2, 5000, 32, 1, 7, dil=13, pad_mode=REFLECT, pre=LEAKY, post=TANH, bias=True),
    "cout1_smem_dil14": _conv(2, 5000, 32, 1, 7, dil=14, pad_mode=REFLECT, pre=LEAKY, post=TANH, bias=True),
    "cout1_stride2": _conv(1, 9000, 32, 1, 7, stride=2, pad=3, pre=RELU, bias=True),
    "cout1_x_off1": _conv(2, 5000, 32, 1, 7, xoff=1, pad_mode=REFLECT, pre=LEAKY, post=TANH, bias=True),
    "cout1_k5_cin2048": _conv(1, 4100, 2048, 1, 5, bias=True),
    "cout1_tiled_lens": _conv(3, 2000, 32, 1, 7, pad_mode=REFLECT, pre=LEAKY, post=TANH, bias=True, lens=(2000, 2, 1)),
    "cout1_lens": _conv(3, 2000, 32, 1, 7, dil=14, pad_mode=REFLECT, pre=LEAKY, bias=True, res="sep", lens=(0, 3, 2000)),
    # ---- split-K edges: M 256 / 257, nk 15 / 16, 16 tiles of 64 x 64 at a budget of 16 / 17 over it, scratch one byte
    # short at 132 SMs (and exactly enough): the room is checked for the 15 splits asked for, before they are evened out to
    # 13 splits of 5 slices
    "split_m256": _dense(256, 1024, 256, bias=True, scratch=1 << 24),
    "split_m257": _dense(257, 1024, 256, bias=True, scratch=1 << 24),
    "split_nk16": _dense(64, 256, 256, bias=True, post=RELU, scratch=1 << 24),
    "split_nk15": _dense(64, 240, 256, bias=True, post=RELU, scratch=1 << 24),
    "split_tiles16": _dense(64, 512, 1024, bias=True, scratch=1 << 24),
    "split_tiles17": _dense(64, 512, 1088, bias=True, scratch=1 << 24),
    "split_scratch_short": _dense(64, 1000, 1024, bias=True, scratch=15 * 64 * 1024 * 4 + 256 - 1),
    "split_scratch_exact": _dense(64, 1000, 1024, bias=True, scratch=15 * 64 * 1024 * 4 + 256),
    # uneven splits: K = 1000 is 63 slices of 16 (the last one 8 wide); 13 splits of 5 at 132 SMs, the last one of 3
    "split_uneven_k1000": _dense(64, 1000, 1024, bias=True, post=LEAKY, acc=True, scale=0.75, scratch=1 << 24),
    "split_uneven_inplace": _dense(5, 1000, 768, bias=True, post=RELU, res="inplace", scratch=1 << 24),
    "split_res_acc_scale": _dense(40, 2048, 384, res="sep", acc=True, scale=1 / 3, pre=LEAKY, scratch=1 << 24),
    # ---- load / store paths on split-K: Cin % 4, Cout % 4, a channel slice, 4-byte offsets of x / y / res, odd ldr
    "split_cin1002": _dense(64, 1002, 256, bias=True, scratch=1 << 24),
    "split_cout1002": _dense(5, 1024, 1002, bias=True, res="sep", scratch=1 << 24),
    "split_ldx_slice": _dense(64, 1024, 512, ldx=1536, xoff=512, bias=True, scratch=1 << 24),
    "split_x_off1": _dense(64, 1024, 512, xoff=1, bias=True, scratch=1 << 24),
    "split_y_off1": _dense(64, 1024, 512, yoff=1, bias=True, acc=True, scratch=1 << 24),
    "split_res_off1": _dense(64, 1024, 512, res="sep", roff=1, scratch=1 << 24),
    "split_ldr_odd": _dense(64, 1024, 512, res="sep", ldr=513, bias=True, scratch=1 << 24),
    # ---- load / store paths on the tiles
    "tile_cin1002": _dense(300, 1002, 256, bias=True),
    "tile_cout130": _conv(2, 500, 64, 130, 3, bias=True, res="sep"),
    "tile_ldx_slice": _dense(300, 1024, 256, ldx=1536, xoff=256, bias=True),
    "tile_x_off1": _conv(2, 150, 64, 96, 3, xoff=1, pad_mode=REFLECT, bias=True),
    "tile_y_off1": _conv(2, 300, 32, 64, 3, yoff=1, bias=True, acc=True),
    "tile128_res_off1": _conv(4, 3900, 16, 128, res="sep", roff=1, scale=0.5),
    "tile_ldr_odd": _conv(2, 500, 40, 32, 3, res="sep", ldr=33, bias=True),
    "tile_inplace_res": _conv(2, 300, 64, 96, 3, pad_mode=REFLECT, res="inplace", bias=True, scale=0.5),
    # ---- the four HiFi-GAN up-samplers, y aligned (vec_y) and 4 bytes off (scalar stores): out_shift < 0, clipped
    "convt_up1": _convt(2, 37, 512, 256, 8),
    "convt_up2": _convt(2, 50, 256, 128, 8),
    "convt_up3": _convt(2, 300, 128, 64, 2),
    "convt_up4": _convt(2, 600, 64, 32, 2),
    "convt_up1_y_off1": _convt(2, 37, 512, 256, 8, yoff=1),
    "convt_up2_y_off1": _convt(2, 50, 256, 128, 8, yoff=1),
    "convt_up3_y_off1": _convt(2, 300, 128, 64, 2, yoff=1),
    "convt_up4_y_off1": _convt(2, 600, 64, 32, 2, yoff=1),
    # ---- geometry: the three paddings with dilation, in_lens of 0, 1, below the halo and Tin
    "pad_zero_dil3": _conv(2, 100, 48, 64, 5, dil=3, bias=True),
    "pad_reflect_dil3": _conv(2, 100, 48, 96, 5, dil=3, pad_mode=REFLECT, pre=LEAKY, bias=True),
    "pad_replicate_dil3": _conv(2, 100, 48, 32, 5, dil=3, pad_mode=REPLICATE, bias=True),
    "lens_reflect": _conv(4, 60, 64, 64, 11, pad_mode=REFLECT, pre=LEAKY, bias=True, lens=(0, 1, 3, 60)),
    "lens_replicate": _conv(4, 60, 32, 130, 5, dil=2, pad_mode=REPLICATE, bias=True, lens=(60, 0, 1, 4)),
    "lens_reflect_m129": _conv(3, 43, 32, 32, 7, dil=2, pad_mode=REFLECT, bias=True, lens=(43, 5, 7)),
}
# the AR decodes' dense layers (causal_step): QKV, out-projection (res == y), FF1 (ReLU), FF2 (res == y)
for _m, (_D, _F) in (("plm", (PLM_D, PLM_F)), ("adm", (ADM_D, ADM_F))):
    for _M in DECODE_ROWS:
        _s = _decode_scratch(_M, _D, _F)
        CASES[f"{_m}_qkv_m{_M}"] = _dense(_M, _D, 3 * _D, bias=True, scratch=_s)
        CASES[f"{_m}_out_m{_M}"] = _dense(_M, _D, _D, bias=True, res="inplace", scratch=_s)
        CASES[f"{_m}_ff1_m{_M}"] = _dense(_M, _D, _F, bias=True, post=RELU, scratch=_s)
        CASES[f"{_m}_ff2_m{_M}"] = _dense(_M, _F, _D, bias=True, res="inplace", scratch=_s)


# ------------------------------------------------------------------------------------------ geometry of a case
@functools.lru_cache(maxsize=None)
def geom(name, B=None):
    """the tap-GEMM a case launches: B, Tin, Tout, Cin, Cout (columns), k, stride, dil, pad, pad_mode, ld / offsets of
    x, y, res, the y batch stride, out_shift, y_batch_elems"""
    c = CASES[name]
    B = c["B"] if B is None else B
    T, Cin, k = c["T"], c["Cin"], c["k"]
    g = dict(B=B, Tin=T, Cin=Cin, k=k, stride=c.get("stride", 1), dil=c.get("dil", 1), pad_mode=c.get("pad_mode", ZERO))
    if "s" in c:
        s, co = c["s"], c["Cout"]
        g.update(Tout=T + 1, Cout=s * co, pad=1, ldy=s * co, ysb=s * T * co, out_shift=-(s // 2) * co, ybe=s * T * co)
    else:
        g["pad"] = c.get("pad", g["dil"] * (k - 1) // 2)
        g["Tout"] = (T + 2 * g["pad"] - g["dil"] * (k - 1) - 1) // g["stride"] + 1
        g["Cout"] = c["Cout"]
        g["ldy"] = c.get("ldy", c["Cout"])
        g.update(ysb=g["Tout"] * g["ldy"], out_shift=0, ybe=0)
    g.update(ldx=c.get("ldx", Cin), xoff=c.get("xoff", 0), yoff=c.get("yoff", 0))
    if c.get("res") == "inplace":
        g.update(ldr=g["ldy"], roff=g["yoff"], rsb=g["ysb"])
    else:
        g.update(ldr=c.get("ldr", g["Cout"]), roff=c.get("roff", 0))
        g["rsb"] = g["Tout"] * g["ldr"]
    return g


def fill_params(name, addr, B=None):
    """mtts_conv_params of case `name` with the buffers at byte addresses addr[x | w | y | res | bias | lens | scratch]
    (element offsets applied here)"""
    c, g = CASES[name], geom(name, B)
    p = L.ConvParams()
    p.x, p.x_batch_stride, p.ldx = addr["x"] + 4 * g["xoff"], g["Tin"] * g["ldx"], g["ldx"]
    p.w, p.bias = addr["w"], addr["bias"] if c.get("bias") else None
    p.y, p.y_batch_stride, p.ldy = addr["y"] + 4 * g["yoff"], g["ysb"], g["ldy"]
    if c.get("res") == "inplace":
        p.res, p.res_batch_stride, p.ldr = p.y, g["ysb"], g["ldy"]
    elif c.get("res"):
        p.res, p.res_batch_stride, p.ldr = addr["res"] + 4 * g["roff"], g["rsb"], g["ldr"]
    p.B, p.Tin, p.Tout, p.Cin, p.Cout = g["B"], g["Tin"], g["Tout"], g["Cin"], g["Cout"]
    p.k, p.stride, p.dil, p.pad, p.pad_mode = g["k"], g["stride"], g["dil"], g["pad"], g["pad_mode"]
    p.pre_act, p.pre_slope = c.get("pre", NONE), PRE_SLOPE
    p.post_act, p.post_slope = c.get("post", NONE), POST_SLOPE
    p.out_scale, p.accumulate = c.get("scale", 1.0), int(bool(c.get("acc")))
    p.out_shift, p.y_batch_elems = g["out_shift"], g["ybe"]
    if c.get("lens"):
        p.in_lens = addr["lens"]
    if c.get("scratch"):
        p.tc_scratch, p.tc_scratch_bytes = addr["scratch"], c["scratch"]
    return p


FAKE = dict(x=1 << 32, w=2 << 32, y=3 << 32, res=4 << 32, bias=5 << 32, lens=6 << 32, scratch=7 << 32)   # 16-byte aligned


def query(p, sms):
    out = (C.c_int32 * 8)()
    L.check(L.lib().mtts_ffma_plan_query(C.byref(p), sms, out))
    return dict(kernel=out[0], BM=out[1], BN=out[2], splits=out[3], kk=out[4], vec_a=out[5], vec_b=out[6], vec_y=out[7])


def plan_of(name, sms, B=None):
    """the plan of case `name` on `sms` SMs with its buffers 16-byte aligned (offsets as the case gives them)"""
    return query(fill_params(name, FAKE, B), sms)


def instantiation(pl):
    return (KERNEL_NAMES[pl["kernel"]], pl["BM"], pl["BN"])


# ------------------------------------------------------------------------------------------ inputs
def _gen(seed):
    g = torch.Generator()
    g.manual_seed(zlib.crc32(seed.encode()))
    return g


@functools.lru_cache(maxsize=8)
def _weights(k, Cin, N, convt_s):
    """packed (k, Cin, N) weights, shared by the cases of one layer shape"""
    g = _gen(f"w{k}x{Cin}x{N}x{convt_s}")
    if convt_s:
        from megatts2_b200 import pack
        w = torch.randn(Cin, N // convt_s, 2 * convt_s, generator=g) / math.sqrt(2 * Cin)
        return pack.pack_conv_transpose(w, torch.zeros(N // convt_s), convt_s)[0].contiguous(), w
    return torch.randn(k, Cin, N, generator=g) / math.sqrt(Cin * k), None


@functools.lru_cache(maxsize=4)
def inputs(name):
    """CPU tensors of case `name`: x (B, Tin, Cin), w (k, Cin, Cout), bias, res (B, Tout, Cout), y0 (B, ysb) - the
    values y holds before the launch (and the residual of an in-place case) - and lens"""
    c, g = CASES[name], geom(name)
    gen = _gen(name)
    d = dict(x=torch.randn(g["B"], g["Tin"], g["Cin"], generator=gen) * 2)
    d["w"], d["w_convt"] = _weights(g["k"], g["Cin"], g["Cout"], c.get("s", 0))
    d["bias"] = torch.randn(g["Cout"], generator=gen) if c.get("bias") else None
    if "s" in c:
        d["b_convt"] = torch.randn(c["Cout"], generator=gen)
        d["bias"] = d["b_convt"].repeat(c["s"])              # pack_conv_transpose: bias tiled s times
    d["res"] = torch.randn(g["B"], g["Tout"], g["Cout"], generator=gen) if c.get("res") == "sep" else None
    d["y0"] = torch.randn(g["B"], g["ysb"], generator=gen)
    d["lens"] = torch.tensor(c["lens"], dtype=torch.int32) if c.get("lens") else None
    return d


def item_inputs(name, b):
    d = inputs(name)
    sl = lambda t: t[b:b + 1] if t is not None else None
    return dict(d, x=sl(d["x"]), res=sl(d["res"]), y0=sl(d["y0"]), lens=sl(d["lens"]))


# ------------------------------------------------------------------------------------------ reference and bar
def _act32(x, a):
    return {NONE: lambda t: t, RELU: F.relu, LEAKY: lambda t: F.leaky_relu(t, PRE_SLOPE)}[a](x)


def row_map(ti, n, mode):
    """input row read for row index ti of an item with n valid rows (-1: zero) - the rule of include/megatts2_b200.h"""
    inside = (ti >= 0) & (ti < n)
    if mode == ZERO:
        return torch.where(inside, ti, -1)
    if mode == REPLICATE:
        r = torch.where(ti < 0, torch.zeros_like(ti), n - 1)
    else:
        r = torch.where(ti < 0, -ti, ti)
        r = torch.where(r >= n, 2 * (n - 1) - r, r)
        r = torch.where((r >= 0) & (r < n), r, -1)
    return torch.where(inside, ti, torch.where(n > 0, r, -1))


def operand_rows(name, d, rows, dev):
    """A (len(rows), k Cin) fp64: the pre-activated input rows each output row m in `rows` multiplies, in the kernel's
    K order (tap j outer, channel c ascending), zero where the input row is outside"""
    g = geom(name, d["x"].shape[0])
    B, Tin, Cin, k = g["B"], g["Tin"], g["Cin"], g["k"]
    x = _act32(d["x"].to(dev), CASES[name].get("pre", NONE)).double()
    x = torch.cat([x.reshape(B * Tin, Cin), torch.zeros(1, Cin, dtype=torch.float64, device=dev)])
    b, t = rows // g["Tout"], rows % g["Tout"]
    n = d["lens"].to(dev).long().clamp(max=Tin)[b] if d["lens"] is not None else torch.full_like(b, Tin)
    ti = t[:, None] * g["stride"] + torch.arange(k, device=dev)[None] * g["dil"] - g["pad"]
    r = row_map(ti, n[:, None], g["pad_mode"])
    idx = torch.where(r >= 0, b[:, None] * Tin + r, B * Tin)
    return x[idx].reshape(len(rows), k * Cin)


def _tf32(t):
    """round-to-nearest-even to TF32's 10 mantissa bits"""
    i = t.float().contiguous().view(torch.int32)
    i = (i + 0xFFF + ((i >> 13) & 1)) & ~0x1FFF
    return i.view(torch.float32)


def chain_rss(A, W, kk):
    """sqrt(sum_i S_i^2) per element of A @ W: S_i the running sums of the kernel's FMA chain (k-major K order, one chain
    per K range of kk 16-channel slices when split, then the reduction's running sums), zero products left out"""
    M, K = A.shape
    N = W.shape[1]
    bounds = list(range(0, K, 16 * kk)) + [K] if kk else [0, K]
    out = torch.empty(M, N, dtype=torch.float64, device=A.device)
    step = max(1, (1 << 26) // (K * N))
    for m0 in range(0, M, step):
        P = A[m0:m0 + step, :, None] * W[None]                     # (rows, K, N) exact products
        ss = torch.zeros(P.shape[0], N, dtype=torch.float64, device=A.device)
        run = torch.zeros_like(ss)
        for z, (lo, hi) in enumerate(zip(bounds[:-1], bounds[1:])):
            S = P[:, lo:hi].cumsum(1)
            ss += (S.square() * (P[:, lo:hi] != 0)).sum(1)
            run = run + S[:, -1]
            if z:
                ss += run.square()
        out[m0:m0 + step] = ss.sqrt()
    return out


def epilogue(name, d, acc, rows, cols, chain):
    """fp64 epilogue of output rows / columns (rows, cols index vectors) over acc (len(rows), len(cols)) with the chain's
    rounding bound; -> (flat positions into the (B, ysb) y buffer, valid mask, values, bars)"""
    c, g = CASES[name], geom(name, d["x"].shape[0])
    dev = acc.device
    b, t = (rows // g["Tout"])[:, None], (rows % g["Tout"])[:, None]
    n = cols[None]
    err = chain.clone()
    v = acc
    if d["bias"] is not None:
        v = v + d["bias"].to(dev).double()[n]
        err = err + U * v.abs()
    post = c.get("post", NONE)
    if post == RELU:
        v = v.clamp_min(0)
    elif post == LEAKY:
        v = torch.where(v > 0, v, v * POST_SLOPE)
        err = err + U * v.abs()
    elif post == TANH:
        v = v.tanh()
        err = err + TANH_ULPS * 2 * U * v.abs()
    y0 = d["y0"].to(dev).double()
    flat = t * g["ldy"] + n + g["out_shift"]
    ybe = g["ybe"] or g["Tout"] * g["ldy"]
    valid = (flat >= 0) & (flat < ybe)
    flat = flat.clamp(0, ybe - 1)
    pos = b * g["ysb"] + flat
    if c.get("res") == "inplace":
        v = v + y0.reshape(-1)[pos]
        err = err + U * v.abs()
    elif c.get("res"):
        v = v + d["res"].to(dev).double()[b, t, n]
        err = err + U * v.abs()
    scale = f32(c.get("scale", 1.0))
    if scale != 1.0:
        v = v * scale
        err = err * abs(scale) + U * v.abs()
    if c.get("acc"):
        v = v + y0.reshape(-1)[pos]
        err = err + U * v.abs()
    return pos, valid, v, err


def reference(name, d, kk, dev, rows=None, cols=None, tf32=False):
    """fp64 values and bars of case `name` (inputs d) at a plan with kk slices per split (0: unsplit), over the given
    output rows / columns (all by default); tf32: the same chain over TF32-rounded x and w"""
    g = geom(name, d["x"].shape[0])
    M = g["B"] * g["Tout"]
    rows = torch.arange(M, device=dev) if rows is None else rows.to(dev)
    cols = torch.arange(g["Cout"], device=dev) if cols is None else cols.to(dev)
    A = operand_rows(name, d, rows, dev)
    W = d["w"].to(dev).reshape(-1, g["Cout"])[:, cols].double()
    if tf32:
        A, W = _tf32(A).double(), _tf32(W).double()
    acc = A @ W
    return epilogue(name, d, acc, rows, cols, LAMBDA * U * chain_rss(A, W, kk))


def full_reference(name, d, kk, dev):
    """the whole y buffer after the launch (fp64) and its per-element bar (0 where the kernel writes nothing)"""
    pos, valid, v, err = reference(name, d, kk, dev)
    y = d["y0"].to(dev).double().reshape(-1).clone()
    bar = torch.zeros_like(y)
    y[pos[valid]] = v[valid]
    bar[pos[valid]] = err[valid]
    return y, bar


# ------------------------------------------------------------------------------------------ one launch
def launch(name, budget, d, B=None):
    """One FFMA tap-GEMM call of case `name` with inputs d under an SM budget -> (the y buffer after it, (B, y batch
    stride), and the plan)"""
    from megatts2_b200 import ops
    c, g = CASES[name], geom(name, B)
    nan = float("nan")
    x = torch.full((g["xoff"] + g["B"] * g["Tin"] * g["ldx"],), nan)
    x[g["xoff"]:].view(g["B"], g["Tin"], g["ldx"])[..., :g["Cin"]] = d["x"]
    y = torch.cat([torch.zeros(g["yoff"]), d["y0"].reshape(-1)])
    bufs = dict(x=x.to(DEV), w=d["w"].to(DEV), y=y.to(DEV))
    if d["bias"] is not None:
        bufs["bias"] = d["bias"].to(DEV)
    if d["res"] is not None:
        r = torch.full((g["roff"] + g["B"] * g["rsb"],), nan)
        r[g["roff"]:].view(g["B"], g["Tout"], g["ldr"])[..., :g["Cout"]] = d["res"]
        bufs["res"] = r.to(DEV)
    if d["lens"] is not None:
        bufs["lens"] = d["lens"].to(DEV)
    if c.get("scratch"):
        bufs["scratch"] = torch.full((c["scratch"],), 255, dtype=torch.uint8, device=DEV)      # NaN floats
    p = fill_params(name, {k: v.data_ptr() for k, v in bufs.items()}, B)
    full = ops.sm_count(torch.device(DEV))
    pl = query(p, budget if 0 < budget < full else full)
    with ops.launch_policy(budget):
        L.check(L.lib().mtts_conv1d_f32(C.byref(p), ops._stream()))
    torch.cuda.synchronize()
    return bufs["y"][g["yoff"]:].view(g["B"], g["ysb"]).cpu(), pl


def run_case(name):
    """Runs case `name` at every budget against fp64, checks equal plans, a repeat and one batch item alone for bit
    identity.  Returns one record per run."""
    from megatts2_b200 import ops
    d = inputs(name)
    full = ops.sm_count(torch.device(DEV))
    refs, seen, records = {}, {}, []
    for budget in BUDGETS:
        sms = budget if 0 < budget < full else full
        y, pl = launch(name, budget, d)
        if pl["kk"] not in refs:
            refs[pl["kk"]] = full_reference(name, d, pl["kk"], DEV)
        ref, bar = refs[pl["kk"]]
        err = (y.reshape(-1).to(DEV).double() - ref).abs()
        bad = ~(err <= bar)                                         # also NaN
        frac = (err / bar.clamp_min(1e-300))[bar > 0].max().item()
        rec = dict(case=name, budget=budget, sms=sms, plan=pl, err_over_bar=frac, max_err=err.max().item())
        records.append(rec)
        print(f"{name:30s} sms {sms:3d}  {instantiation(pl)} splits {pl['splits']:2d} kk {pl['kk']:2d} "
              f"vec {pl['vec_a']}{pl['vec_b']}{pl['vec_y']}  err {frac:.3f} of the bar")
        assert not bad.any(), (rec, int(bad.sum()), int(bad.nonzero()[0]))
        key = tuple(sorted(pl.items()))
        if key in seen:
            assert torch.equal(y, seen[key]), f"{rec}: not bit-identical to an earlier run of the same plan"
        seen[key] = y
    assert torch.equal(launch(name, 0, d)[0], y), f"{name}: a repeat launch is not bit-identical"
    # one batch item alone against its rows of the batched launch (unsplit: the same FMA chain whatever the kernel)
    g = geom(name)
    if g["B"] > 1:
        b = g["B"] - 1
        for budget in (1, 0):
            y_all, pl_all = launch(name, budget, d)
            y_one, pl_one = launch(name, budget, item_inputs(name, b), B=1)
            if SPLITK in (pl_all["kernel"], pl_one["kernel"]):
                continue
            assert torch.equal(y_one[0], y_all[b]), f"{name} item {b} @{budget}: {pl_one} alone vs {pl_all} batched"
    return records


# ------------------------------------------------------------------------------------------ GPU: the table
@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(CASES))
def test_ffma_plans_vs_fp64(name):
    import helpers
    for rec in run_case(name):
        helpers.record("ffma_plans", rec)


@gpu
def test_ops_conv1d_stride_and_in_lens():
    """ops.conv1d's plumbing of stride, padding, in_lens and a channel-sliced input view (FFMA engine: no w_tc)"""
    from megatts2_b200 import ops
    g = _gen("ops_conv1d")
    x = torch.randn(3, 41, 48, generator=g)
    w = torch.randn(3, 24, 20, generator=g) / math.sqrt(72)
    lens = torch.tensor([41, 9, 20], dtype=torch.int32)
    xs = x[..., 8:32]
    y = ops.conv1d(xs.to(DEV), w.to(DEV), None, k=3, stride=2, pad=1, in_lens=lens.to(DEV)).cpu()
    assert y.shape == (3, 21, 20)
    for b in range(3):
        xb = xs[b:b + 1].clone()
        xb[:, int(lens[b]):] = 0                                  # rows past the item's length read as zero
        ref = F.conv1d(xb.transpose(1, 2).double(), w.permute(2, 1, 0).double(), stride=2, padding=1)
        assert (y[b].double() - ref.transpose(1, 2)[0]).abs().max().item() < 1e-5


# ------------------------------------------------------------------------------------------ CPU: plans, bar
def _edge(name, sms=H100_SMS, **kw):
    pl = plan_of(name, sms)
    want = dict(pl, **kw)
    assert pl == want, (name, sms, pl, kw)


def test_plan_query_pins_routing_edges():
    """mtts_ffma_plan_query (host only) at the dispatch edges of conv1d_ffma()"""
    _edge("cout32", kernel=TILE, BM=128, BN=32)
    _edge("cout33", kernel=TILE, BM=128, BN=64, vec_b=0, vec_y=0)
    _edge("cout64", kernel=TILE, BM=128, BN=64)
    _edge("cout65", kernel=TILE, BM=64, BN=64, vec_b=0, vec_y=0)
    _edge("tiles128_119", kernel=TILE, BM=64, BN=64)
    _edge("tiles128_120", kernel=TILE, BM=128, BN=128)
    _edge("cout1_m4095", kernel=TILE, BM=128, BN=32)
    _edge("cout1_m4096", kernel=COUT1_TILED, BM=256, BN=1)
    _edge("cout1_cin128", kernel=COUT1)                   # Cin <= 128, but the tiled window needs 135 KB
    _edge("cout1_cin132", kernel=COUT1)
    _edge("cout1_smem_dil13", kernel=COUT1_TILED)
    _edge("cout1_smem_dil14", kernel=COUT1)
    _edge("cout1_stride2", kernel=COUT1)
    _edge("cout1_x_off1", kernel=TILE, BM=128, BN=32, vec_a=0)
    _edge("cout1_k5_cin2048", kernel=TILE, BM=128, BN=32)
    _edge("cout1_tiled_lens", kernel=COUT1_TILED)
    _edge("cout1_lens", kernel=COUT1)
    assert plan_of("cout1_tiled_lens", H100_SMS, B=1)["kernel"] == TILE          # one item alone: M = 2000 < 4096
    # split-K
    _edge("split_m256", kernel=SPLITK, BM=64, BN=64, splits=16, kk=4)
    _edge("split_m257", kernel=TILE, BM=64, BN=64, splits=1, kk=0)
    _edge("split_nk16", kernel=SPLITK, splits=4, kk=4)
    _edge("split_nk15", kernel=TILE, BM=64, BN=64, splits=1, kk=0)
    _edge("split_tiles16", 16, kernel=SPLITK, splits=2, kk=16)
    _edge("split_tiles17", 16, kernel=TILE)
    _edge("split_tiles17", 100, kernel=SPLITK)
    _edge("split_scratch_short", kernel=TILE, BM=64, BN=64)
    _edge("split_scratch_short", 100, kernel=SPLITK, splits=11, kk=6)
    _edge("split_scratch_exact", kernel=SPLITK, splits=13, kk=5)
    _edge("split_uneven_k1000", kernel=SPLITK, splits=13, kk=5)   # 63 slices: 12 x 5 + 3
    for sms in (1, 3):
        assert plan_of("split_uneven_k1000", sms)["kernel"] == TILE
    # load / store paths of the split
    _edge("split_cin1002", kernel=SPLITK, vec_a=0, vec_b=1, vec_y=1)
    _edge("split_cout1002", kernel=SPLITK, vec_a=1, vec_b=0, vec_y=0)
    _edge("split_x_off1", kernel=SPLITK, vec_a=0)
    _edge("split_y_off1", kernel=SPLITK, vec_y=0)
    _edge("split_res_off1", kernel=SPLITK, vec_y=0)
    _edge("split_ldr_odd", kernel=SPLITK, vec_y=0)
    _edge("split_ldx_slice", kernel=SPLITK, vec_a=1)
    # the transposed-conv form: never split, never a Cout = 1 kernel; vec_y follows y's alignment
    for s in ("convt_up1", "convt_up2", "convt_up3", "convt_up4"):
        assert plan_of(s, H100_SMS)["vec_y"] == 1 and plan_of(s + "_y_off1", H100_SMS)["vec_y"] == 0
    # the decode's layers split K while the batch is small
    assert plan_of("plm_ff2_m1", H100_SMS)["kernel"] == SPLITK and plan_of("plm_ff1_m200", H100_SMS)["kernel"] == TILE


def test_plan_query_checks_and_empty_calls():
    """the query's argument checks and error codes are those of the launch; no output rows -> MTTS_FFMA_NONE"""
    out = (C.c_int32 * 8)()
    lib = L.lib()
    assert lib.mtts_ffma_plan_query(None, H100_SMS, out) == BAD_ARG
    p = fill_params("cout32", FAKE)
    assert lib.mtts_ffma_plan_query(C.byref(p), 0, out) == BAD_ARG
    for field, bad in (("x", None), ("Cin", 0), ("k", 0), ("stride", 0), ("pad_mode", 3), ("ldx", 47)):
        q = fill_params("cout32", FAKE)
        setattr(q, field, bad)
        assert lib.mtts_ffma_plan_query(C.byref(q), H100_SMS, out) == BAD_ARG, field
        assert lib.mtts_conv1d_f32(C.byref(q), None) == BAD_ARG, field
    q = fill_params("cout32", FAKE)
    q.Tout = 0
    assert query(q, H100_SMS)["kernel"] == FFMA_NONE


def test_table_reaches_every_kernel():
    """The table's plans at budgets 1, 3, 16, 100 and 132 SMs launch every kernel and tile conv1d_ffma() has and no other,
    with vec_a, vec_b and vec_y each on and off on the tiles and on split-K"""
    reached, flags = set(), {}
    for name in CASES:
        for sms in (1, 3, 16, 100, H100_SMS):
            pl = plan_of(name, sms)
            reached.add(instantiation(pl))
            fam = "splitk" if pl["kernel"] == SPLITK else "tile" if pl["kernel"] == TILE else "cout1"
            for v in ("vec_a", "vec_b", "vec_y"):
                flags.setdefault((fam, v), set()).add(pl[v])
            if pl["kernel"] == SPLITK:
                assert 2 <= pl["splits"] <= 16 and (pl["splits"] - 1) * pl["kk"] < -(-CASES[name]["Cin"] // 16)
    want = {("tile", 128, 32), ("tile", 128, 64), ("tile", 128, 128), ("tile", 64, 64), ("splitk", 64, 64),
            ("cout1", 256, 1), ("cout1_tiled", 256, 1)}
    assert reached == want, (sorted(want - reached), sorted(reached - want))
    for fam in ("tile", "splitk"):
        for v in ("vec_a", "vec_b", "vec_y"):
            assert flags[(fam, v)] == {0, 1}, (fam, v)


def test_transposed_conv_form_is_conv_transpose1d():
    """The contract the reference restates (a 2-tap conv over s Cout columns written at out_shift and clipped to the
    y_batch_elems) computes F.conv_transpose1d at the four HiFi-GAN up-sampler shapes"""
    for name in ("convt_up1", "convt_up2", "convt_up3", "convt_up4"):
        c, d = CASES[name], inputs(name)
        s, co = c["s"], c["Cout"]
        y, bar = full_reference(name, d, 0, "cpu")
        ref = F.conv_transpose1d(_act32(d["x"], LEAKY).transpose(1, 2).double(), d["w_convt"].double(),
                                 d["b_convt"].double(), stride=s, padding=s // 2).transpose(1, 2)
        assert (bar > 0).sum() == ref.numel()
        assert (y.view(c["B"], -1) - ref.reshape(c["B"], -1)).abs().max().item() < 1e-12, name


def _sample(n, m):
    return torch.linspace(0, n - 1, min(n, m)).round().long().unique()


def test_bar_rejects_tf32():
    """The bar has teeth: on sampled elements of every case, at every split its plans take, the same chain over
    TF32-rounded x and w misses the bar by at least 4x"""
    worst = {}
    for name in CASES:
        g = geom(name)
        d = inputs(name)
        rows, cols = _sample(g["B"] * g["Tout"], 12), _sample(g["Cout"], 12)
        for kk in sorted({plan_of(name, s)["kk"] for s in (1, 3, 16, 100, H100_SMS)}):
            _, valid, v, bar = reference(name, d, kk, "cpu", rows, cols)
            _, _, v32, _ = reference(name, d, kk, "cpu", rows, cols, tf32=True)
            diff = (v32 - v).abs()[valid]
            if diff.max() == 0:
                continue
            ratio = (diff / bar[valid])[diff > 0].max().item()   # rows of zero input (outside every item) are exact
            worst[(name, kk)] = ratio
            assert ratio >= TEETH, (name, kk, ratio)
    print("smallest TF32 miss / bar:", min(worst.values()))
