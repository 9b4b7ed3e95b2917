"""fp64 reference of the mel front end (mtts_mel_spectrogram_f32, csrc/mel.cu) and the per-element error bar of its fp32
kernel.

    out[b, m, f] = log(max(sum_k fb[k, m] |X_b,f[k]|, clamp)),   X_b,f = rfft(w * x_b[256 f - 512 : 256 f + 512])

x_b is clip b's first L_b samples, reflect-padded by 512 at both ends (torch.stft(center=True)); f < 1 + L_b / 256.  The
reference starts from the exact fp32 samples, window and dense fp32 filterbank, and the fp32 value of clamp, promoted to
fp64.

The bar.  u = 2^-24, N = 1024.  Per frame, with p = x w (the frame's windowed samples, exact):

  products   the kernel rounds each x_n (w_n / 2) once (the 1/2 of the packed-real split rides on the window, exactly),
             and the untangle doubles them back: every bin is off by at most u ||p||_1.
  FFT        the 512-point complex transform Z of the packed pairs is three radix-8 Stockham passes, each a diagonal of
             twiddles then 8-point DFTs: a scaled unitary map, so an error of relative size eta in one pass's outputs
             (in the 2-norm) reaches Z as eta ||Z||_2, and the passes add.  Per 8-point DFT: three levels of complex adds
             (u each) and, in the first, the (1 -+ i) / sqrt 2 rotations (one more add, the product and the rounded
             constant: 3u more), 6u.  A twiddle is rounded per component (u) and multiplied in real arithmetic (sqrt 5 u,
             which also covers a contracted FMA form); the third pass's upper half multiplies two rounded twiddles first
             ((2 + sqrt 5) u).  Passes: 6u, (1 + sqrt 5 + 6) u, (2 + 2 sqrt 5 + 6) u; 27.7u in all.
             The untangle forms X_k = (1 - i w^k) Z_k + (1 + i w^k) conj Z_512-k, whose coefficients have squared moduli
             summing to 4, so an error in Z reaches any one bin at most doubled (Cauchy-Schwarz).  Its own roundings:
             u |E| for E = a + conj c, (2 + sqrt 5) u |O| for O = (a - conj c) / i times the rounded w^k, and u |X_k|
             for the last add; |E|, |O| <= sqrt 2 ||Z||_2 and |X_k| <= 2 ||Z||_2 give 9.4u ||Z||_2.  Together
             64.8u ||Z||_2, and ||Z||_2 = sqrt(N / 8) ||p||_2 (Parseval), so every bin is off by at most
             C_FFT u sqrt(N) ||p||_2 with C_FFT = 64.8 / sqrt 8 = 22.9.  This is a worst case for one bin: the 2-norm of
             the whole error vector may sit in it.
  magnitude  |X_k| = sqrt.approx(re^2 + im^2): the sum of squares (two roundings) then sqrt.approx (relative error
             2^-23, PTX ISA): 3u |X_k|.
  filterbank four FMA chains per mel, tap t into partial sum t mod 4 (the bands start on a multiple of 4 bins, so that
             is bin k mod 4), in bin order, then (a0 + a1) + (a2 + a3).  Each FMA rounds its running sum S once; FMAs
             with a zero weight are exact.  So u sum S over the taps with a nonzero weight, plus 2u acc for the two levels
             of adds (all terms are non-negative), plus the bin errors above weighted by the bank column.
  log        out = __logf(max(mel, clamp)).  fmaxf is 1-Lipschitz, so a mel error d maps to the interval
             [log max(mel - d, clamp), log max(mel + d, clamp)] around log max(mel, clamp); the bar takes its larger
             side (first order: d / max(mel, clamp)).  ASSUMED from the CUDA C Programming Guide (intrinsic functions):
             __logf is within 2^-21.41 absolute for arguments in [0.5, 2] and within 3 ulp otherwise; the bar adds both,
             2^-21.41 + 6u |out|.
  infinities clamp = 0 on a band with no energy gives -inf, which must match the reference exactly.

Bins 40-80 dB below the frame's energy get a bar set by that energy: the FFT term is per frame, not per bin.  Loud bands
get a bar of a few u in the log domain."""
import math
import os
import re

import numpy as np

U = 2.0 ** -24
N_FFT, HOP, N_BINS = 1024, 256, 513
C_FFT = (2 * (6 + (1 + math.sqrt(5) + 6) + (2 + 2 * math.sqrt(5) + 6))
         + math.sqrt(2) * (1 + 2 + math.sqrt(5)) + 2) / math.sqrt(8)
LOG_ABS = 2.0 ** -21.41

MEL_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "megatts2_b200", "csrc", "mel.cu")


def kernel_constants(path=MEL_CU):
    """the integer constexprs of mel.cu (MEL_FBW, MEL_SPAN, MEL_FPB, MEL_HOP, ...), evaluated from the source"""
    env = {}
    for decl in re.findall(r"^constexpr int ([^;]+);", open(path).read(), flags=re.M):
        for part in decl.split(","):
            name, expr = (s.strip() for s in part.split("=", 1))
            env[name] = int(eval(expr, {"__builtins__": {}}, dict(env)))
    return env


# ------------------------------------------------------------------------------------------ filterbanks
def unpack_grouped(fb_w, fb_off, fb_start, n_mels, n_bins=N_BINS):
    """the grouped banded form pack_grouped_filterbank writes -> the dense (n_bins, n_mels) bank it stands for; checks
    the layout rules of the header on the way (aligned starts, reads below bin n_bins + 3, empty slots past n_mels)"""
    limit = (n_bins + 3) // 4 * 4
    G = (n_mels + 3) // 4
    assert len(fb_off) == G + 1 and len(fb_start) == 4 * G and fb_off[0] == 0 and len(fb_w) == fb_off[G]
    dense = np.zeros((limit, n_mels), dtype=np.float32)
    for g in range(G):
        block = np.asarray(fb_w[fb_off[g]:fb_off[g + 1]]).reshape(4, -1)
        ln = block.shape[1]
        assert ln % 4 == 0
        for i in range(4):
            m, s0 = 4 * g + i, int(fb_start[4 * g + i])
            assert s0 % 4 == 0 and s0 + ln <= limit
            if m < n_mels:
                dense[s0:s0 + ln, m] += block[i]
            else:
                assert not block[i].any()
    assert not dense[n_bins:].any()
    return dense[:n_bins]


def chain_counts(fb):
    """cnt[k, m]: the nonzero taps of mel m at bins k' >= k with k' = k mod 4, i.e. the FMAs of k's partial sum whose
    running sum contains bin k's product"""
    n_bins, M = fb.shape
    limit = (n_bins + 3) // 4 * 4
    nz = np.zeros((limit, M))
    nz[:n_bins] = fb != 0
    r = nz.reshape(limit // 4, 4, M)
    return r[::-1].cumsum(0)[::-1].reshape(limit, M)[:n_bins]


# ------------------------------------------------------------------------------------------ the reference
def frames(x, pad="reflect"):
    """(L,) -> (1 + L / 256, 1024) frames of the padded clip"""
    L = x.shape[0]
    xp = np.pad(x, N_FFT // 2, mode=pad)
    idx = np.arange(1 + L // HOP)[:, None] * HOP + np.arange(N_FFT)[None, :]
    return xp[idx]


def clip_mel(x, window, fb, clamp, *, pad="reflect", rfft=None, dtype=np.float64, bar=False):
    """one clip (L,) fp32 -> (n_mels, F) in `dtype`, and its bar when asked.  pad / rfft / dtype exist for the wrong
    variants and the fp32 restatements the tests build on the same pipeline."""
    fr = frames(np.asarray(x, dtype=dtype), pad) * np.asarray(window, dtype=dtype)
    X = (rfft or np.fft.rfft)(fr, axis=-1)
    mag = np.abs(X).astype(dtype)
    fbd = np.asarray(fb, dtype=dtype)
    mel = mag @ fbd
    cl = dtype(np.float32(clamp))
    with np.errstate(divide="ignore"):
        out = np.log(np.maximum(mel, cl))
    if not bar:
        return out.T
    E = U * np.abs(fr).sum(-1) + C_FFT * U * math.sqrt(N_FFT) * np.sqrt(np.square(fr).sum(-1))       # (F,)
    d = (E[:, None] + 3 * U * mag) @ fbd + U * (mag @ (fbd * chain_counts(fb))) + 2 * U * mel
    M = np.maximum(mel, cl)
    with np.errstate(divide="ignore", invalid="ignore"):
        up = np.log(np.maximum(mel + d, cl)) - out
        down = out - np.log(np.maximum(mel - d, cl))
    b = np.maximum(up, down) + LOG_ABS + 6 * U * np.abs(np.where(np.isfinite(out), out, 0.0))
    b = np.where(M > 0, b, 0.0)                        # -inf in the reference: the kernel must match it exactly
    return out.T, b.T


def reference(wav, lens, window, fb, clamp, **kw):
    """wav (B, L_max) fp32, lens None or per-clip lengths (clamped to L_max, as the kernel does) -> out, bar
    (B, n_mels, 1 + L_max / 256) fp64; frames a clip does not have are NaN"""
    B, L_max = wav.shape
    F = 1 + L_max // HOP
    out = np.full((B, fb.shape[1], F), np.nan)
    bar = np.full_like(out, np.nan)
    for b in range(B):
        Lb = L_max if lens is None else min(int(lens[b]), L_max)
        o, e = clip_mel(wav[b, :Lb], window, fb, clamp, bar=True, **kw)
        out[b, :, :o.shape[1]], bar[b, :, :o.shape[1]] = o, e
    return out, bar


def spectrogram(wav, lens, window, fb, clamp, **kw):
    """the same pipeline without the bar (the wrong variants and the fp32 restatement)"""
    B, L_max = wav.shape
    out = np.full((B, fb.shape[1], 1 + L_max // HOP), np.nan)
    for b in range(B):
        Lb = L_max if lens is None else min(int(lens[b]), L_max)
        o = clip_mel(wav[b, :Lb], window, fb, clamp, **kw)
        out[b, :, :o.shape[1]] = o
    return out


def excess(out, ref, bar):
    """per element: error / bar (0 on the frames the reference does not have).  Infinities must match exactly (0 if they
    do, inf if not)."""
    out = np.asarray(out, np.float64)
    have = ~np.isnan(ref)
    inf = have & (~np.isfinite(ref) | ~np.isfinite(out))
    fin = have & ~inf
    r = np.zeros(ref.shape)
    r[inf] = np.where(out[inf] == ref[inf], 0.0, np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        r[fin] = np.abs(out[fin] - ref[fin]) / bar[fin]
    r[np.isnan(r)] = 0.0                               # 0 / 0: an exact match where the bar is 0
    return r
