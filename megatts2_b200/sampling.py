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
    >= 0 and every row with a positive fp32 sum."""
    if not bool(torch.isfinite(w64).all()) or bool((w64 < 0).any()):
        raise L.MttsError(f"{what}: every weight must be finite and >= 0")
    w32 = w64.to(torch.float32).contiguous()
    s = w32.sum(-1)
    if not bool(torch.isfinite(s).all()) or bool((s <= 0).any()):
        raise L.MttsError(f"{what}: every weight row needs a positive, finite sum")
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
