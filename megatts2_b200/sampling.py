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
