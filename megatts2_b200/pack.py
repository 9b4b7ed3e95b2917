"""One-time weight re-layout for the tap-GEMM kernels (host-side plumbing, torch ops).

The kernels take weights as (k, Cin, Cout) row-major ("tap-major, output-channel
contiguous"); torch stores nn.Linear as (N, K), nn.Conv1d as (Cout, Cin, k) and
nn.ConvTranspose1d as (Cin, Cout, k).
"""
import ctypes as C

import torch

from . import _lib as L


FMT_BF16X3, FMT_F16X2, FMT_F16 = 0, 1, 2
F16X2_SCALE = 2048.0


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _permute_copy(src, dst, B, T, Cc, sx, sy):
    """dst[b, t, c] (element strides sy) = src[b, t, c] (element strides sx) through the library's tiled copy kernel
    (coalesced on both sides): every device-side weight re-layout is ONE launch of a product kernel."""
    L.check(L.lib().mtts_copy_strided_f32(C.c_void_p(src.data_ptr()), sx[0], sx[1], sx[2], C.c_void_p(dst.data_ptr()),
                                          sy[0], sy[1], sy[2], B, T, Cc, 0, _stream()))
    return dst


def _f32(w):
    w = w.detach()
    return w if w.dtype == torch.float32 else w.float()


def pack_linear(w):
    """nn.Linear weight (N, K) -> (1, K, N)."""
    w = _f32(w)
    if not w.is_cuda:
        return w.t().contiguous().unsqueeze(0)
    N, K = w.shape
    out = torch.empty(1, K, N, dtype=torch.float32, device=w.device)
    return _permute_copy(w, out, 1, K, N, (0, w.stride(1), w.stride(0)), (0, N, 1))


def pack_conv(w):
    """nn.Conv1d weight (Cout, Cin, k) -> (k, Cin, Cout)."""
    w = _f32(w)
    if not w.is_cuda:
        return w.permute(2, 1, 0).contiguous()
    co, ci, k = w.shape
    out = torch.empty(k, ci, co, dtype=torch.float32, device=w.device)
    return _permute_copy(w, out, k, ci, co, (w.stride(2), w.stride(1), w.stride(0)), (ci * co, co, 1))


def pack_qkv(wq, wk, wv):
    """three (D, D) projections -> (1, D, 3D) so one GEMM yields [q | k | v]."""
    ws = [_f32(wq), _f32(wk), _f32(wv)]
    if not ws[0].is_cuda:
        return pack_linear(torch.cat(ws, 0))
    N, K = ws[0].shape
    out = torch.empty(1, K, 3 * N, dtype=torch.float32, device=ws[0].device)
    for i, w in enumerate(ws):
        _permute_copy(w, out[:, :, i * N:], 1, K, N, (0, w.stride(1), w.stride(0)), (0, 3 * N, 1))
    return out


def cat_vectors(*vs):
    """concatenate 1-D fp32 parameters (bias packing) - with the library's copy kernel on the device"""
    vs = [_f32(v) for v in vs]
    if not vs[0].is_cuda:
        return torch.cat(vs).contiguous()
    out = torch.empty(sum(v.numel() for v in vs), dtype=torch.float32, device=vs[0].device)
    o = 0
    for v in vs:
        _permute_copy(v, out[o:], 1, 1, v.numel(), (0, 0, v.stride(0)), (0, 0, 1))
        o += v.numel()
    return out


def pack_conv_transpose(w, bias, stride):
    """nn.ConvTranspose1d weight (Cin, Cout, k = 2*stride), padding (k - stride)//2, as the
    2-tap conv the kernel runs:  super-row u: out[u*s + r - pad] = x[u-1] W[..., r+s] + x[u] W[..., r]
    -> weight (2, Cin, s*Cout) with column index r*Cout + co, bias tiled s times."""
    cin, cout, k = w.shape
    s = stride
    assert k == 2 * s, "only kernel == 2*stride transposed convs are on the path (HiFi-GAN V1)"
    w = _f32(w)
    if not w.is_cuda:
        tap0 = w[:, :, s:].permute(0, 2, 1).reshape(cin, s * cout)   # pairs with x[u-1]
        tap1 = w[:, :, :s].permute(0, 2, 1).reshape(cin, s * cout)   # pairs with x[u]
        wp = torch.stack([tap0, tap1], 0).contiguous()
        bp = _f32(bias).repeat(s).contiguous() if bias is not None else None
        return wp, bp
    wp = torch.empty(2, cin, s * cout, dtype=torch.float32, device=w.device)
    sx = (w.stride(0), w.stride(2), w.stride(1))                     # (ci, r, co) walk of the source
    _permute_copy(w[:, :, s:], wp[0], cin, s, cout, sx, (s * cout, cout, 1))
    _permute_copy(w[:, :, :s], wp[1], cin, s, cout, sx, (s * cout, cout, 1))
    bp = None
    if bias is not None:
        b = _f32(bias)
        bp = torch.empty(s * cout, dtype=torch.float32, device=w.device)
        _permute_copy(b, bp, 1, s, cout, (0, 0, b.stride(0)), (0, cout, 1))
    return wp, bp


def cat_rows(*ws):
    """stack (N_i, K) fp32 matrices along rows -> (sum N_i, K), device copies through the library's kernel"""
    ws = [_f32(w) for w in ws]
    if not ws[0].is_cuda:
        return torch.cat(ws, 0).contiguous()
    K = ws[0].shape[1]
    out = torch.empty(sum(w.shape[0] for w in ws), K, dtype=torch.float32, device=ws[0].device)
    o = 0
    for w in ws:
        _permute_copy(w, out[o:], 1, w.shape[0], K, (0, w.stride(0), w.stride(1)), (0, K, 1))
        o += w.shape[0]
    return out


def plane_dtype(fmt):
    return torch.bfloat16 if fmt == FMT_BF16X3 else torch.float16


def pack_tc_planes(w, fmt=FMT_BF16X3):
    """(N, K) fp32 weight -> tensor-core operand planes, the same split the kernels apply to activations
    (a format has 3 - fmt planes):
    bf16x3: (3, N, K) bf16 with w = w1 + w2 + w3 to ~2^-24 (round-to-nearest at every step);
    f16x2:  (2, N, K) fp16 with w = w1 + w2 * 2^-11 (the residual is stored scaled by 2^11);
    f16:    (1, N, K) fp16 with w ~ fp16(w) (round-to-nearest; half precision, not fp32-grade)."""
    w = _f32(w)
    if w.is_cuda:
        if not w.is_contiguous():
            w = w.contiguous()
        N, K = w.shape
        out = torch.empty(3 - fmt, N, K, dtype=plane_dtype(fmt), device=w.device)
        L.check(L.lib().mtts_split_planes_f32(C.c_void_p(w.data_ptr()), K, N, K, C.c_void_p(out.data_ptr()), fmt, _stream()))
        return out
    if fmt == FMT_F16:
        return w.to(torch.float16)[None]
    if fmt == FMT_F16X2:
        p1 = w.to(torch.float16)
        p2 = ((w - p1.float()) * F16X2_SCALE).to(torch.float16)
        return torch.stack([p1, p2], 0).contiguous()
    p1 = w.to(torch.bfloat16)
    r1 = w - p1.float()
    p2 = r1.to(torch.bfloat16)
    p3 = (r1 - p2.float()).to(torch.bfloat16)
    return torch.stack([p1, p2, p3], 0).contiguous()


def pack_conv_tc_planes(w, fmt=FMT_BF16X3):
    """nn.Conv1d weight (Cout, Cin, k) fp32 -> (3 | 2 | 1, k, Cout, Cin) operand planes (per-tap K-major B operands)."""
    w = _f32(w)
    co, ci, k = w.shape
    if w.is_cuda:
        tmp = torch.empty(k, co, ci, dtype=torch.float32, device=w.device)
        _permute_copy(w, tmp, k, co, ci, (w.stride(2), w.stride(0), w.stride(1)), (co * ci, ci, 1))
        flat = tmp.view(k * co, ci)
    else:
        flat = w.permute(2, 0, 1).contiguous().reshape(-1, ci)
    return pack_tc_planes(flat, fmt).reshape(-1, k, co, ci)


def pack_conv_transpose_tc_planes(wp, fmt=FMT_BF16X3):
    """packed transposed-conv weight (2, Cin, s*Cout) fp32 -> (3 | 2 | 1, 2, s*Cout, Cin) operand planes."""
    two, cin, n = wp.shape
    if wp.is_cuda:
        tmp = torch.empty(two, n, cin, dtype=torch.float32, device=wp.device)
        _permute_copy(wp, tmp, two, n, cin, (wp.stride(0), wp.stride(2), wp.stride(1)), (n * cin, cin, 1))
        flat = tmp.view(two * n, cin)
    else:
        flat = wp.permute(0, 2, 1).reshape(-1, cin)
    return pack_tc_planes(flat, fmt).reshape(-1, two, n, cin)


ENGINE_FFMA, ENGINE_BF16X3, ENGINE_F16X2, ENGINE_F16 = 0, 1, 2, 3


_engine_override = None


class engine_scope:
    """``with pack.engine_scope(pack.ENGINE_BF16X3): ...`` - every module whose ``.engine`` attribute is unset uses this
    engine inside the block (plans are keyed by engine, so they rebuild on entry and again on exit)."""

    def __init__(self, engine):
        self.engine = engine

    def __enter__(self):
        global _engine_override
        self.prev, _engine_override = _engine_override, self.engine
        return self

    def __exit__(self, *exc):
        global _engine_override
        _engine_override = self.prev
        return False


def default_engine() -> int:
    """Engine for the dense contractions with M >= 128 (MEGATTS2_ENGINE = f16x2 | bf16x3 | ffma | f16):
    2 = wgmma with f16x2 operands (default: 3 MMAs per fp32-grade product, |activation| <= 65504 guarded by the
    overflow flag, see ops.tc_overflow; at the low end an operand keeps |x - x^| <= 2^-22 |x| + 2^-36, so values
    below 2^-14 lose precision and values below about 2^-35 vanish - training therefore runs on bf16x3), 1 = wgmma
    with bf16x3 operands (6 MMAs, full fp32 range), 0 = fp32 FFMA everywhere.  These three are fp32-grade at
    activation magnitudes; ids are bit-identical between them in the tests.  Attention runs on the f16x2 tensor-core
    kernel only under engines 2 and 3; under 1 and 0 it stays on the fp32 kernel.
    3 = wgmma with f16 operands is NOT: the opt-in half-precision inference engine (one fp16 plane per operand, one MMA
    per product into an fp32 accumulator, the same fp16 range guard).  Its results differ from the others by fp16
    rounding, and ids may differ too; it is reported separately."""
    import os
    if _engine_override is not None:
        return _engine_override
    v = os.environ.get("MEGATTS2_ENGINE", "f16x2").lower()
    if v in ("ffma", "fp32", "0"):
        return ENGINE_FFMA
    if v in ("bf16x3", "tc", "1"):
        return ENGINE_BF16X3
    if v in ("f16", "3"):
        return ENGINE_F16
    return ENGINE_F16X2


def engine_fmt(engine: int) -> int:
    return {ENGINE_F16X2: FMT_F16X2, ENGINE_F16: FMT_F16}.get(engine, FMT_BF16X3)


_epoch = 0


def invalidate_plans():
    """Force every cached weight plan to be rebuilt on its next use.  ``signature`` sees in-place updates made through
    autograd-visible ops (``p.add_()``, ``load_state_dict``, optimiser steps); writes through ``param.data`` or
    ``torch.no_grad`` views that bypass the version counter need this call."""
    global _epoch
    _epoch += 1


def signature(tensors):
    """Cheap change detector for a parameter set (storage address + in-place version + invalidation epoch)."""
    return tuple((t.data_ptr(), t._version) for t in tensors) + (_epoch,)




def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class PlanMixin:
    """nn.Module mixin: the cached plan holds ctypes structs (raw device pointers) that must
    not be pickled / deep-copied with the module; it is rebuilt lazily instead."""

    def __getstate__(self):
        d = self.__dict__.copy()
        d["_plan"] = None
        d.pop("_graph_caches", None)
        return d

    def _graphs(self, name="main"):
        """CUDA-graph cache ``name`` of this module's device-only drivers (megatts2_b200/graphs.py).  Each name is a cache
        of its own, so one kind of call never evicts another's graphs."""
        caches = self.__dict__.setdefault("_graph_caches", {})
        if name not in caches:
            from . import graphs
            caches[name] = graphs.GraphedCall()
        return caches[name]


class Plan:
    """Keeps packed device tensors and the ctypes structs that point at them alive together."""

    _serial = 0

    def __init__(self):
        self.keep = []
        self.sig = None
        Plan._serial += 1
        self.serial = Plan._serial          # identifies THIS packing in graph-cache keys (id() values get reused)

    def hold(self, t):
        self.keep.append(t)
        return t

    def p(self, t):
        """hold a tensor and return its device pointer as an int (for ctypes struct fields)."""
        if t is None:
            return None
        t = t.detach()
        if t.dtype != torch.float32 or not t.is_contiguous():
            t = t.float().contiguous()
        self.keep.append(t)
        return t.data_ptr()


def build_encoder_struct(plan, layers, d_model, n_heads, ff_dim, conv_ff, engine=0):
    """layers: iterable of objects with .norm1 .norm2 .attn(w_q,w_k,w_v,out_proj[0]) .ff"""
    arr = (L.EncoderLayer * len(layers))()
    tc = engine >= 1
    fmt = engine_fmt(engine)

    def tcc(w):
        t = pack_conv_tc_planes(w, fmt)
        plan.keep.append(t)
        return t.data_ptr()

    def tcp(w):
        t = pack_tc_planes(w, fmt)
        plan.keep.append(t)
        return t.data_ptr()
    for i, lyr in enumerate(layers):
        a = lyr.attn
        e = arr[i]
        e.ln1_g, e.ln1_b = plan.p(lyr.norm1.weight), plan.p(lyr.norm1.bias)
        e.ln2_g, e.ln2_b = plan.p(lyr.norm2.weight), plan.p(lyr.norm2.bias)
        e.w_qkv = plan.p(pack_qkv(a.w_q.weight, a.w_k.weight, a.w_v.weight))
        e.b_qkv = plan.p(cat_vectors(a.w_q.bias, a.w_k.bias, a.w_v.bias))
        e.w_o, e.b_o = plan.p(pack_linear(a.out_proj[0].weight)), plan.p(a.out_proj[0].bias)
        if conv_ff:
            e.w_ff1, e.b_ff1 = plan.p(pack_conv(lyr.ff[0].weight)), plan.p(lyr.ff[0].bias)
            e.w_ff2, e.b_ff2 = plan.p(pack_conv(lyr.ff[2].weight)), plan.p(lyr.ff[2].bias)
        else:
            e.w_ff1, e.b_ff1 = plan.p(pack_linear(lyr.ff[0].weight)), plan.p(lyr.ff[0].bias)
            e.w_ff2, e.b_ff2 = plan.p(pack_linear(lyr.ff[3].weight)), plan.p(lyr.ff[3].bias)
        if tc:
            e.w_qkv_tc = tcp(cat_rows(a.w_q.weight, a.w_k.weight, a.w_v.weight))
            e.w_o_tc = tcp(a.out_proj[0].weight)
            if conv_ff:
                e.w_ff1_tc, e.w_ff2_tc = tcc(lyr.ff[0].weight), tcc(lyr.ff[2].weight)
            else:
                e.w_ff1_tc, e.w_ff2_tc = tcp(lyr.ff[0].weight), tcp(lyr.ff[3].weight)
    plan.hold(arr)
    enc = L.Encoder()
    enc.n_layers, enc.d_model, enc.n_heads, enc.ff_dim, enc.conv_ff = len(layers), d_model, n_heads, ff_dim, int(conv_ff)
    enc.engine = int(engine) if tc else 0
    enc.layers = C.cast(arr, C.POINTER(L.EncoderLayer))
    return enc


def fill_conv_blocks(plan, arr, offset, stack, engine=0):
    """stack: ResidualBlockStack; writes n_stacks*n_blocks mtts_conv_block entries at arr[offset:]."""
    i = offset
    for cs in stack.conv_stacks:
        for blk in cs.blocks:
            arr[i].w, arr[i].b = plan.p(pack_conv(blk.conv.weight)), plan.p(blk.conv.bias)
            arr[i].ln_g, arr[i].ln_b = plan.p(blk.norm.weight), plan.p(blk.norm.bias)
            if engine >= 1:
                t = pack_conv_tc_planes(blk.conv.weight, engine_fmt(engine))
                plan.keep.append(t)
                arr[i].w_tc = t.data_ptr()
            i += 1
    return i
