"""Opt-in sampling of the prosody LM's decode (``MegaPLM.infer`` / ``infer_causal``, ``Megatts.synthesize``).

``Sampling`` holds the parameters of one call; passing ``sampling=None`` (the default everywhere) keeps the greedy decode.
Each step's code is drawn on the device (include/megatts2_b200.h, ``mtts_sampling``): temperature, then top-k, then
top-p, then a Gumbel-max draw whose noise depends only on (seed, row key, step, token).  So a draw does not depend on the
batch a row runs in, and several takes of one utterance are the same row under different keys."""
import ctypes as C
import dataclasses
import math
import numbers

import torch

from . import _lib as L


def _f32(v):
    return C.c_float(v).value


@dataclasses.dataclass(frozen=True)
class Sampling:
    """temperature: y = logits / temperature (0 = greedy); top_k: keep the k most likely codes (0 = off); top_p: keep the
    shortest most-likely prefix with probability mass >= top_p (1 = off); seed: 64-bit seed of the noise.  temperature
    and top_p are used as fp32 numbers."""
    temperature: float = 1.0
    top_k: int = 0
    top_p: float = 1.0
    seed: int = 0

    def __post_init__(self):
        def real(name, v):
            if isinstance(v, bool) or not isinstance(v, numbers.Real):
                raise L.MttsError(f"Sampling.{name} must be a real number, got {v!r}")
            return float(v)

        def integer(name, v):
            if isinstance(v, bool) or not isinstance(v, numbers.Integral):
                raise L.MttsError(f"Sampling.{name} must be an integer, got {v!r}")
            return int(v)

        t, p = real("temperature", self.temperature), real("top_p", self.top_p)
        k, s = integer("top_k", self.top_k), integer("seed", self.seed)
        if not (math.isfinite(t) and t >= 0.0 and math.isfinite(_f32(t))):
            raise L.MttsError(f"Sampling.temperature must be finite and >= 0, got {t}")
        if not 0 <= k < 2 ** 31:
            raise L.MttsError(f"Sampling.top_k must be >= 0, got {k}")
        if not (0.0 < _f32(p) <= 1.0):
            raise L.MttsError(f"Sampling.top_p must be in (0, 1], got {p}")
        if not 0 <= s < 2 ** 64:
            raise L.MttsError(f"Sampling.seed must be in [0, 2**64), got {s}")
        for name, v in (("temperature", t), ("top_k", k), ("top_p", p), ("seed", s)):
            object.__setattr__(self, name, v)

    def graph_key(self):
        """The parameters a captured decode bakes in (the seed and the keys are device inputs instead)."""
        return (_f32(self.temperature), self.top_k, _f32(self.top_p))

    def seed_tensor(self, device):
        """The seed as a 1-element int64 device tensor (its bits are the uint64 seed)."""
        s = self.seed - 2 ** 64 if self.seed >= 2 ** 63 else self.seed
        return torch.tensor([s], dtype=torch.int64, device=device)

    def struct(self, seed, keys):
        """ctypes ``mtts_sampling`` over device tensors ``seed`` (1,) and ``keys`` (rows,) int64."""
        return L.Sampling(_f32(self.temperature), self.top_k, _f32(self.top_p), 0, seed.data_ptr(), keys.data_ptr())


MIX_MAX_SOURCES = 8


def _real_weights(weights, what, shapes):
    """``weights`` as a tensor of real numbers (not yet checked for shape or values)."""
    try:
        w = torch.as_tensor(weights).detach()
    except (TypeError, ValueError, RuntimeError) as e:
        raise L.MttsError(f"{what}: weights must be a {shapes} array of real numbers ({e})") from None
    if w.dtype == torch.bool or w.is_complex() or not (w.is_floating_point() or w.dtype in (
            torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8)):
        raise L.MttsError(f"{what}: weights must be real numbers, got {w.dtype}")
    return w


def _checked_rows(w64, what):
    """fp64 weights whose last dim is one weight row -> the rows as a contiguous fp32 tensor, every weight finite and
    >= 0 and every row with a positive fp32 sum.  An error names the first bad weight or row by its index."""
    bad = ~torch.isfinite(w64) | (w64 < 0)
    if bool(bad.any()):
        i = tuple(int(x) for x in bad.nonzero()[0])
        raise L.MttsError(f"{what}: weight {list(i)} = {float(w64[i])}: every weight must be finite and >= 0")
    w32 = w64.to(torch.float32).contiguous()
    s = w32.sum(-1)
    bad = ~torch.isfinite(s) | (s <= 0)
    if bool(bad.any()):
        r = tuple(int(x) for x in bad.nonzero()[0])
        raise L.MttsError(f"{what}: weight row {list(r)} sums to {float(s[r])}: every weight row needs a positive, finite "
                          "sum")
    return w32


def mix_weights(weights, K, B, what="prosody mix"):
    """The mix weights of ``MegaPLM.infer_mix`` and ``MegaADM.infer_mix`` as a validated (B, K) fp32 CPU tensor:
    ``weights`` is (K,) (the same row for every utterance) or (B, K); every weight finite and >= 0, every row with a
    positive fp32 sum.  ``what`` names the mix in the error messages."""
    if not 1 <= K <= MIX_MAX_SOURCES:
        raise L.MttsError(f"{what}: K = {K} sources, expected 1 to {MIX_MAX_SOURCES}")
    w = _real_weights(weights, what, "(K,) or (B, K)")
    w64 = w.to(device="cpu", dtype=torch.float64)
    if w64.dim() == 1:
        w64 = w64.unsqueeze(0).expand(B, -1)
    if tuple(w64.shape) != (B, K):
        raise L.MttsError(f"{what}: weights of shape {tuple(w.shape)}, expected ({K},) or ({B}, {K})")
    return _checked_rows(w64, what)


def per_step(weights):
    """Whether mix weights are a schedule, (B, T, K) with one row per step, rather than one row per utterance."""
    try:
        return torch.as_tensor(weights).dim() == 3
    except (TypeError, ValueError, RuntimeError):
        return False


def mix_step_weights(weights, K, B, T, what="prosody mix"):
    """Mix weights that change along the utterance as a validated (B, T, K) fp32 CPU tensor: row (b, t) weighs the K
    sources at step t of utterance b, under ``mix_weights``'s rules for each row."""
    if not 1 <= K <= MIX_MAX_SOURCES:
        raise L.MttsError(f"{what}: K = {K} sources, expected 1 to {MIX_MAX_SOURCES}")
    w = _real_weights(weights, what, "(B, T, K)")
    if tuple(w.shape) != (B, T, K):
        raise L.MttsError(f"{what}: weights of shape {tuple(w.shape)}, expected ({B}, {T}, {K}) (one row per step)")
    return _checked_rows(w.to(device="cpu", dtype=torch.float64), what)


def synth_mix_weights(weights, K, B, Tp, what):
    """The validated (B, K) CPU weights of a synthesis mix over Tp phones, or (B, Tp, K) when ``weights`` has one row
    per phone."""
    if per_step(weights):
        return mix_step_weights(weights, K, B, Tp, what)
    return mix_weights(weights, K, B, what)


DURATION_MAX = 128          # the ADM's durations are 1..128 frames
PIN_MAX = 127               # the reference's ADM never trains on a duration >= 128
FIT_MAX_PHONES = 8192       # mtts_fit_durations_f32's bound on Tp


def _integers(v, what, shapes):
    """``v`` as an int64 CPU tensor (the one device-to-host read when ``v`` is a device tensor)."""
    try:
        t = torch.as_tensor(v).detach()
    except (TypeError, ValueError, RuntimeError) as e:
        raise L.MttsError(f"{what}: expected a {shapes} array of integers ({e})") from None
    if t.dtype not in (torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8):
        raise L.MttsError(f"{what}: expected integers, got {t.dtype}")
    return t.to(device="cpu", dtype=torch.int64)


def duration_scale(scale, B, Tp):
    """``duration_scale`` as a validated fp32 CPU tensor: () (one value), (B,) (one per utterance) or (B, Tp) (one per
    phone), every value finite and > 0 as an fp32 number.  Above 1 the utterance is slower."""
    if isinstance(scale, bool):
        raise L.MttsError(f"duration_scale must be a real number or a tensor of them, got {scale!r}")
    s = _real_weights(scale, "duration_scale", "(), (B,) or (B, Tp)").to(device="cpu", dtype=torch.float64)
    if tuple(s.shape) not in ((), (B,), (B, Tp)):
        raise L.MttsError(f"duration_scale: shape {tuple(s.shape)}, expected (), ({B},) or ({B}, {Tp})")
    s32 = s.to(torch.float32)
    if not bool(torch.isfinite(s32).all()) or bool((s32 <= 0).any()):
        raise L.MttsError("duration_scale: every value must be finite and > 0 (as an fp32 number)")
    return s32.contiguous()


def pinned_durations(pinned, B, Tp):
    """``pinned_durations`` as a validated (B, Tp) int32 CPU tensor: -1 leaves a phone free, 1..127 pins it to that many
    frames (the range the ADM is trained on)."""
    p = _integers(pinned, "pinned_durations", "(B, Tp)")
    if tuple(p.shape) != (B, Tp):
        raise L.MttsError(f"pinned_durations: shape {tuple(p.shape)}, expected ({B}, {Tp})")
    bad = (p != -1) & ((p < 1) | (p > PIN_MAX))
    if bool(bad.any()):
        b, i = (int(x) for x in bad.nonzero()[0])
        raise L.MttsError(f"pinned_durations[{b}, {i}] = {int(p[b, i])}: expected -1 (free) or 1..{PIN_MAX}")
    return p.to(torch.int32).contiguous()


def pinned_codes(pinned, B, T, V):
    """``pinned`` prosody codes as a validated (B, T) int32 CPU tensor: -1 leaves step j of utterance b free, 0..V-1 fixes
    its code.  Anything else (BOS = V and pad = V + 1 included) is an error: a pin is a code the model emits."""
    p = _integers(pinned, "pinned codes", "(B, T)")
    if tuple(p.shape) != (B, T):
        raise L.MttsError(f"pinned codes: shape {tuple(p.shape)}, expected ({B}, {T})")
    bad = (p != -1) & ((p < 0) | (p >= V))
    if bool(bad.any()):
        b, j = (int(x) for x in bad.nonzero()[0])
        raise L.MttsError(f"pinned codes[{b}, {j}] = {int(p[b, j])}: expected -1 (free) or 0..{V - 1}")
    return p.to(torch.int32).contiguous()


def pinned_runs(pins, return_logits=False):
    """The maximal runs [j0, j1) of steps at which some row of the validated (B, T) ``pins`` is free: the steps a pinned
    decode enqueues.  A step pinned in every row is never read back (step j reads codes < j only), so it is skipped;
    ``return_logits`` keeps the single run [0, T) so every step's logits exist."""
    T = pins.shape[1]
    if return_logits:
        return ((0, T),) if T else ()
    free = (pins < 0).any(0).tolist() if pins.shape[0] else [False] * T
    runs, j = [], 0
    while j < T:
        if not free[j]:
            j += 1
            continue
        j0 = j
        while j < T and free[j]:
            j += 1
        runs.append((j0, j))
    return tuple(runs)


def total_frames(total, B, Tp, pinned=None):
    """``total_frames`` as a validated (B,) int32 CPU tensor, each total feasible for its utterance: with F its free
    phones (all phones without ``pinned``, a validated (B, Tp) tensor) and P the sum of its pins, [|F| + P, 128 |F| + P]."""
    t = _integers(total, "total_frames", "(B,)")
    if tuple(t.shape) != (B,):
        raise L.MttsError(f"total_frames: shape {tuple(t.shape)}, expected ({B},)")
    pins = pinned.to(torch.int64) if pinned is not None else torch.full((B, Tp), -1, dtype=torch.int64)
    free = (pins < 1).sum(1)
    psum = pins.clamp(min=0).sum(1)
    lo, hi = free + psum, DURATION_MAX * free + psum
    for b in range(B):
        if not int(lo[b]) <= int(t[b]) <= int(hi[b]):
            raise L.MttsError(f"total_frames[{b}] = {int(t[b])} is outside utterance {b}'s feasible range "
                              f"[{int(lo[b])}, {int(hi[b])}] ({int(free[b])} free phones, {int(psum[b])} pinned frames)")
    return t.to(torch.int32).contiguous()


def duration_control(scale, total, pinned, B, Tp):
    """The validated (scale, total, pinned) CPU tensors of a duration-controlled call (each None when not given)."""
    pins = None if pinned is None else pinned_durations(pinned, B, Tp)
    if (scale is not None or total is not None) and Tp > FIT_MAX_PHONES:
        raise L.MttsError(f"duration_scale / total_frames: Tp = {Tp} phones is above the bound of {FIT_MAX_PHONES}")
    sc = None if scale is None else duration_scale(scale, B, Tp)
    tot = None if total is None else total_frames(total, B, Tp, pins)
    return sc, tot, pins


def row_keys(keys, rows, device):
    """Per-row 64-bit keys as a contiguous (rows,) int64 device tensor; None -> arange(rows)."""
    if keys is None:
        return torch.arange(rows, dtype=torch.int64, device=device)
    k = torch.as_tensor(keys)
    if k.dtype not in (torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8):
        raise L.MttsError(f"keys: expected an integer tensor, got {k.dtype}")
    if k.shape != (rows,):
        raise L.MttsError(f"keys: expected shape ({rows},), got {tuple(k.shape)}")
    return k.to(device=device, dtype=torch.int64).contiguous()
