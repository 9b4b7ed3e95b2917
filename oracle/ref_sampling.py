"""numpy restatement of the opt-in PLM sampler (include/megatts2_b200.h, mtts_sampling) - the ORACLE of
megatts2_b200/csrc/sample.cu.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) - never imported by the product.

Philox4x32-10 in exact uint32 arithmetic; y = z / temperature in fp32 (as the device divides); the filters, the softmax
and the Gumbel scores in fp64."""
import numpy as np
import torch

from . import ref_megatts2 as R

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr (..., 4), key (..., 2) unsigned 32-bit words -> (..., 4) uint32 (Salmon et al., SC'11; Random123 constants)."""
    c = [np.asarray(ctr, dtype=np.uint64)[..., j] & MASK for j in range(4)]
    k = [np.asarray(key, dtype=np.uint64)[..., j] & MASK for j in range(2)]
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]                    # exact: both factors < 2**32
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & MASK, p1 >> np.uint64(32), p1 & MASK
        c = [hi1 ^ c[1] ^ k[0], lo1, hi0 ^ c[3] ^ k[1], lo0]
        k = [(k[0] + W0) & MASK, (k[1] + W1) & MASK]
    return np.stack(c, -1).astype(np.uint32)


def words(seed, key, step, idx):
    """Philox word of token idx (array) at AR step `step` for row key `key` under `seed` (64-bit integers)."""
    idx = np.asarray(idx, dtype=np.uint64)
    seed, key = int(seed) % 2 ** 64, int(key) % 2 ** 64
    ctr = np.stack(np.broadcast_arrays(idx >> np.uint64(2), np.uint64(step), np.uint64(key & 0xFFFFFFFF),
                                       np.uint64(key >> 32)), -1)
    kk = np.broadcast_to(np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64), ctr.shape[:-1] + (2,))
    r = philox4x32_10(ctr, kk)
    return np.take_along_axis(r, (idx & np.uint64(3)).astype(np.int64)[..., None], -1)[..., 0]


def gumbel(w):
    """-log(-log u), u = ((w >> 8) + 0.5) * 2^-24, in fp64 (1 - u exact for the upper half)."""
    m = (np.asarray(w, dtype=np.uint64) >> np.uint64(8)).astype(np.float64)
    e = np.where(m < 2 ** 23, -np.log((m + 0.5) * 2.0 ** -24), -np.log1p(-((2 ** 24 - 1 - m) + 0.5) * 2.0 ** -24))
    return -np.log(e)


def tempered(z, temperature):
    """y = z / temperature in fp32, widened to fp64."""
    z = np.asarray(z, dtype=np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return (z / np.float32(temperature)).astype(np.float64)


def kept_set(y, top_k, top_p):
    """Indices of the candidates kept by top-k and top-p, in (value descending, index ascending) order, and their softmax
    weights exp(y - y_max) (fp64).  y has no +inf here."""
    V = y.shape[0]
    cand = np.nonzero(~np.isnan(y) & (y != -np.inf))[0]
    order = cand[np.lexsort((cand, -y[cand]))]
    if 0 < top_k < V:
        order = order[:top_k]
    e = np.exp(y[order] - y[order[0]]) if order.size else np.zeros(0)
    p = float(np.float32(top_p))
    if p < 1.0 and order.size:
        cum = np.cumsum(e)
        c = int(np.argmax(cum >= p * cum[-1])) + 1
        order, e = order[:c], e[:c]
    return order, e


def sample_row(z, step, temperature, top_k, top_p, seed, key):
    """The contract for one row -> (pick, scores of the kept tokens (fp64, aligned with `kept`), kept indices).
    Greedy cases return (argmax, None, None)."""
    z = np.asarray(z, dtype=np.float32)
    if float(np.float32(temperature)) == 0.0 or top_k == 1:
        return greedy(z), None, None
    y = tempered(z, temperature)
    inf = np.nonzero(y == np.inf)[0]
    if inf.size:
        return int(inf[0]), None, None
    kept, _ = kept_set(y, top_k, top_p)
    if kept.size == 0:
        return 0, None, None
    s = y[kept] + gumbel(words(seed, key, step, kept))
    best = s.max()
    return int(kept[s == best].min()), s, kept


def greedy(z):
    """argmax_rows: the first maximum, NaN never a candidate, 0 for a row without a candidate."""
    z = np.asarray(z, dtype=np.float32)
    ok = ~np.isnan(z) & (z != -np.inf)
    if not ok.any():
        return 0
    m = z[ok].max()
    return int(np.nonzero(ok & (z == m))[0][0])


def sample_rows(logits, step, temperature, top_k, top_p, seed, keys):
    """logits (rows, V) -> (picks (rows,) int64, relative gap of the two best fp64 scores per row (inf when the pick is
    not a score contest))."""
    logits = np.asarray(logits, dtype=np.float32)
    picks = np.zeros(logits.shape[0], dtype=np.int64)
    gaps = np.full(logits.shape[0], np.inf)
    for r in range(logits.shape[0]):
        picks[r], s, _ = sample_row(logits[r], step, temperature, top_k, top_p, seed, int(keys[r]))
        if s is not None and s.size > 1:
            top2 = np.sort(s)[-2:]
            gaps[r] = (top2[1] - top2[0]) / max(1.0, abs(top2[1]))
    return picks, gaps


def target_distribution(z, temperature, top_k, top_p):
    """The fp64 probability of each token under the contract (softmax of the kept tokens; Gumbel-max theorem)."""
    y = tempered(z, temperature)
    kept, e = kept_set(y, top_k, top_p)
    p = np.zeros(y.shape[0])
    p[kept] = e / e.sum()
    return p


def plm_infer_sampled(sd, tc_latent, cfg, temperature, top_k, top_p, seed, keys, return_logits=False):
    """MegaPLM.infer (models/megatts2.py:165-181) with each step's code drawn by the sampler instead of the argmax."""
    B, T, _ = tc_latent.shape
    codes = torch.full((B, 1), cfg["vq_bins"], dtype=torch.int64)
    all_logits = []
    for t in range(T):
        lg = R.plm_step_logits(sd, tc_latent, codes, cfg)
        all_logits.append(lg)
        picks, _ = sample_rows(lg.numpy(), t, temperature, top_k, top_p, seed, keys)
        codes = torch.cat([codes, torch.from_numpy(picks)[:, None]], 1)
    out = codes[:, 1:]
    return (out, torch.stack(all_logits, 1)) if return_logits else out
