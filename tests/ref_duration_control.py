"""Restatements of duration control (include/megatts2_b200.h, mtts_fit_durations_f32 and mtts_adm_infer_pinned_f32) - the
oracles of fit_durations_kernel (csrc/ops.cu) and of MegaADM.infer / infer_mix with ``pinned``.

Test infrastructure only.  The fit compares candidates as rationals: w_i / (k + 1/2) against w_j / (m + 1/2) as
``Fraction``s, never in floating point.  To stay fast at Tp = 8192, ``fit`` uses fp64 values only to narrow the search:
every candidate whose fp64 value lies within a relative 1e-9 of the approximate N-th largest is ordered exactly, and the
ones outside that window differ from it by far more than fp64's rounding (2^-53 relative), so their side is certain.
``fit_brute`` sorts every candidate exactly; the CPU tests check that the two agree."""
from fractions import Fraction

import numpy as np
import torch

import ref_duration_mix as DM

MAX_D = 128            # durations are 1..128 frames
EXTRA = MAX_D - 1      # candidates per free phone: the frames above its first
WINDOW = 1e-9


def weights(raw, scale=None):
    """w = fl32(raw * scale) (numpy broadcasting), with NaN, +-inf and w <= 0 counted as 0."""
    raw = np.asarray(raw, np.float32)
    c = np.float32(1.0) if scale is None else np.asarray(scale, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        w = (raw * c).astype(np.float32)
    return np.where(np.isfinite(w) & (w > 0), w, np.float32(0.0)).astype(np.float32)


def round_rule(w):
    """The no-total rule: clamp(trunc(fl32(w + 0.5)), 1, 128) for w >= 0 (adm_finalize's rounding)."""
    v = (np.asarray(w, np.float32) + np.float32(0.5)).astype(np.float32)
    return np.clip(np.trunc(np.minimum(v, np.float32(4 * MAX_D))).astype(np.int64), 1, MAX_D)


def _value(w, k):
    """Candidate k (1-based) of a phone of weight w, exactly."""
    return Fraction(float(w)) * 2 / (2 * k + 1)


def _row(w, pins, L, top):
    Tp = len(w)
    pins = np.full(Tp, -1, np.int64) if pins is None else np.asarray(pins, np.int64)
    free = pins < 1
    d = np.where(free, 0, pins).astype(np.int64)
    if L is None:
        d[free] = round_rule(w[free])
        return d
    idx = np.nonzero(free)[0]
    N = int(L) - int(pins[~free].sum()) - len(idx)
    assert 0 <= N <= EXTRA * len(idx), (L, N, len(idx))
    d[idx] = 1
    if N:
        for c in top(w[idx], N):                 # flat candidate numbers c = j * EXTRA + (k - 1) over the free phones
            d[idx[c // EXTRA]] += 1
    return d


def _top_brute(wf, N):
    cands = [(-_value(wf[j], k), j, j * EXTRA + k - 1) for j in range(len(wf)) for k in range(1, EXTRA + 1)]
    cands.sort(key=lambda t: (t[0], t[1]))
    return [c for _, _, c in cands[:N]]


def _top_window(wf, N):
    v = (wf.astype(np.float64)[:, None] / (np.arange(1, EXTRA + 1, dtype=np.float64) + 0.5)[None, :]).ravel()
    t = np.partition(v, v.size - N)[v.size - N]
    sure = np.nonzero(v > t * (1 + WINDOW))[0]
    window = np.nonzero(np.abs(v - t) <= t * WINDOW)[0]
    assert len(sure) < N <= len(sure) + len(window)
    order = sorted(window, key=lambda c: (-_value(wf[c // EXTRA], c % EXTRA + 1), c // EXTRA))
    return list(sure) + order[:N - len(sure)]


def _fit(raw, scale, total, pinned, top):
    raw = np.asarray(raw, np.float32)
    B, Tp = raw.shape
    sc = None if scale is None else np.broadcast_to(np.asarray(scale, np.float32).reshape(
        {0: (1, 1), 1: (B, 1), 2: (B, Tp)}[np.ndim(scale)]), (B, Tp))
    w = weights(raw, sc)
    out = np.empty((B, Tp), np.int64)
    for b in range(B):
        out[b] = _row(w[b], None if pinned is None else np.asarray(pinned)[b],
                      None if total is None else int(np.asarray(total)[b]), top)
    return torch.from_numpy(out.astype(np.int32))


def fit(raw, scale=None, total=None, pinned=None):
    """ops.fit_durations: raw (B, Tp), scale None / scalar / (B,) / (B, Tp), total None / (B,), pinned None / (B, Tp)
    (-1 free) -> (B, Tp) int32."""
    return _fit(raw, scale, total, pinned, _top_window)


def fit_brute(raw, scale=None, total=None, pinned=None):
    """``fit`` with every candidate sorted exactly (small inputs only)."""
    return _fit(raw, scale, total, pinned, _top_brute)


def adm_infer_pinned(sd, tc_latents, cfg, weights_, pinned, return_raw=False):
    """MegaADM.infer_mix (K = 1 with weight 1: MegaADM.infer) with pins teacher-forced: ref_duration_mix.adm_infer_mix's
    loop, where step t feeds back pinned[b, t] instead of the mixed readout when that pin is >= 1.  weights_ (B, K) fp32,
    pinned (B, T).  -> durations (B, T, 1) int32 [, raw (B, T, 1), raw_src (K, B, T)]."""
    K = len(tc_latents)
    B, T, _ = tc_latents[0].shape
    dtype = tc_latents[0].dtype
    w = np.asarray(weights_, dtype=np.float32).reshape(B, K)
    pins = np.asarray(pinned, np.int64).reshape(B, T)
    p = torch.zeros(B, 1, 1, dtype=dtype)
    raw_src = torch.full((K, B, T), float("nan"), dtype=dtype)
    for t in range(T):
        ys = {}
        for k in range(K):
            if return_raw or bool((w[:, k] > 0).any()):
                ys[k] = DM.adm_step(sd, tc_latents[k], p, t, cfg)[:, 0, 0]
                raw_src[k, :, t] = ys[k]
        r = torch.zeros(B, dtype=dtype)
        for b in range(B):
            if pins[b, t] >= 1:
                r[b] = float(pins[b, t])
                continue
            yb = torch.stack([ys[k][b] if k in ys else torch.zeros((), dtype=dtype) for k in range(K)])
            r[b] = DM.mix_readout(yb, w[b])
        p = torch.cat([p, r.reshape(B, 1, 1)], 1)
    raw = p[:, 1:, :]
    dur = (raw + 0.5).to(torch.int32).clamp(1, 128)
    return (dur, raw, raw_src) if return_raw else dur
