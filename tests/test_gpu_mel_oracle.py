"""The mel front end (mel_kernel, csrc/mel.cu) against fp64, at every window, filterbank, staging path, clip edge and
output layout mtts_mel_spectrogram_f32 / _ragged_f32 accept.  The reference and its per-element bar are in ref_mel.py,
whose docstring derives the bar.

Paths, per CTA of 16 frames (mirrored in `paths`, with the kernel's constants read from mel.cu):
  filterbank   staged in shared memory when the packed bank has at most MEL_FBW floats (Slaney 80: 1344), else read
               from global memory (Slaney 128: 1584; n_mels 1, 6 and 127; wide custom banks)
  staging      float4 loads on interior tiles (16-byte aligned wav and row stride, no reflection in the 4864-sample
               span), scalar with reflection elsewhere: edge tiles, and every tile of a misaligned or odd-stride wav
  descriptors  n_mels not a multiple of 4 leaves slots with mel index -1
  store order  frames fast (out_sf <= out_sm) or mels fast; padded strides on both
  lengths      ragged clips (each with its own reflection and frame count; lens[b] > L_max is clamped), frame counts at
               the 16-frame tile edge, clips of 513..1025 samples whose frames reflect at both ends

Signals are chosen for what white noise cannot show: tones on and between bins, at the untangle's special bins (0, 256,
512) and at lane boundaries; impulses at the clip's ends and on hop boundaries; silence; int16-scale and near-floor
amplitudes; an 80 dB mixture.  Bin probes (one-hot banks, 5 of them cover bins 0..512 with every start alignment) check
the 513 magnitudes of every frame directly.

The CPU tests at the top check the reference and its bar: an fp32 restatement (scipy's fp32 FFT) and the fp32
torch.stft oracle stay within it, five plausible wrong front ends miss it by at least 4x, and the case table reaches
every path.  The GPU tests compare every case with the bar, and check bit for bit what must not depend on the launch: a
repeat, the batch around a clip, the staging path, the filterbank path, the output layout and the B > 65535 fold.
Frames a clip does not have, and every byte of a padded output outside the tensor, must keep a sentinel."""
import functools
import math
import zlib

import numpy as np
import pytest
import scipy.fft
import torch

import helpers
import ref_mel as RM
from megatts2_b200 import _lib as LIB
from megatts2_b200.modules.tokenizer import pack_grouped_filterbank, slaney_mel_filterbank

DEV = "cuda"
gpu = pytest.mark.gpu
K = RM.kernel_constants()
FBW, FPB, HOP, SPAN = K["MEL_FBW"], K["MEL_FPB"], K["MEL_HOP"], K["MEL_SPAN"]
SENTINEL = -12345.5


# ------------------------------------------------------------------------------------------ inputs
@functools.lru_cache(maxsize=None)
def window(kind):
    n = np.arange(1024, dtype=np.float64)
    if kind == "hann":                                  # the product table: torch.hann_window(1024), periodic
        return torch.hann_window(1024, dtype=torch.float32).numpy()
    if kind == "hamming":                               # w[0] = 0.08: sample 0 of every frame counts
        return (0.54 - 0.46 * np.cos(2 * np.pi * n / 1024)).astype(np.float32)
    assert kind == "rand"                               # positive and asymmetric
    return np.random.default_rng(7).uniform(0.05, 1.0, 1024).astype(np.float32)


def _wide_bands(n, seed, min_len=150):
    rng = np.random.default_rng(seed)
    fb = np.zeros((513, n), dtype=np.float32)
    for m in range(n):
        lo = int(rng.integers(0, 513 - min_len))
        hi = int(rng.integers(lo + min_len, 514))
        fb[lo:hi, m] = rng.uniform(0.01, 1.0, hi - lo)
    return fb


@functools.lru_cache(maxsize=None)
def bank(name):
    """(dense (513, n_mels) fp32, fb_w, fb_off, fb_start)"""
    if name.startswith("slaney"):
        fb = slaney_mel_filterbank(n_mels=int(name[6:]))
    elif name.startswith("probe"):                      # mel m selects bin 5 m + j alone, with weight 1
        j = int(name[5:])
        bins = np.arange(j, 513, 5)
        fb = np.zeros((513, len(bins)), dtype=np.float32)
        fb[bins, np.arange(len(bins))] = 1.0
    elif name == "wide":
        fb = _wide_bands(24, 11)
    else:
        assert name == "mixed128"                       # Slaney 80, then 48 wide bands: the same groups 0..19, global
        fb = np.concatenate([slaney_mel_filterbank(n_mels=80), _wide_bands(48, 12, 60)], 1)
    return (fb,) + pack_grouped_filterbank(fb)


def signal(kind, n, rng):
    t = np.arange(n, dtype=np.float64)
    ph = rng.uniform(0, 2 * np.pi)
    tone = lambda k, a=0.5: a * np.sin(2 * np.pi * k * t / 1024 + rng.uniform(0, 2 * np.pi))   # noqa: E731
    if kind == "noise":
        return rng.uniform(-1, 1, n)
    if kind == "tone_centre":
        return tone(37.0)
    if kind == "tone_half":
        return tone(37.5)
    if kind == "tone_dc":
        return np.full(n, 0.5)
    if kind == "tone_256":
        return 0.5 * np.cos(np.pi * t / 2 + ph)
    if kind == "tone_nyq":
        return 0.5 * np.cos(np.pi * t)
    if kind == "tone_lanes":
        return sum(tone(k, 0.2) for k in (31, 32, 255, 257))
    if kind == "chirp":
        return 0.7 * np.sin(2 * np.pi * 0.5 * t * t / (2 * n) + ph)
    if kind == "impulses":
        x = np.zeros(n)
        x[HOP::HOP] = 0.5
        x[0], x[n - 1] = 1.0, -0.8
        return x
    if kind == "silence":
        return np.zeros(n)
    if kind == "silence_tiny":
        x = np.zeros(n)
        x[n // 2 + 3] = 1e-4
        return x
    if kind == "dc_offset":
        return 0.25 + 1e-3 * rng.uniform(-1, 1, n)
    if kind == "int16":
        x = rng.integers(-32768, 32768, n).astype(np.float64)
        x[0], x[n // 2], x[n - 1] = -32768, 32767, -32768
        return x
    if kind == "floor":                                 # mels near the 1e-5 clamp
        return 2e-5 * rng.uniform(-1, 1, n)
    assert kind == "mixture"                            # 0, -40 and -80 dB
    return tone(20.3, 1.0) + tone(101.7, 1e-2) + tone(333.2, 1e-4)


SIGNALS = ("noise", "tone_centre", "tone_half", "tone_dc", "tone_256", "tone_nyq", "tone_lanes", "chirp", "impulses",
           "silence", "silence_tiny", "dc_offset", "int16", "floor", "mixture")


# ------------------------------------------------------------------------------------------ case table
def _case(block, sig, L, lens=None, win="hann", bank="slaney80", clamp=1e-5, lay="mm", align="vec"):
    return dict(block=block, sig=sig, L=L, lens=tuple(lens) if lens else None, win=win, bank=bank, clamp=clamp,
                lay=lay, align=align)


def _cases():
    out = []
    lays, aligns = ("mm", "fm", "pad", "padfm"), ("vec", "vec", "mis", "odd")
    # ---- signals on the product configuration, long enough for interior tiles
    for i, s in enumerate(SIGNALS):
        out.append(_case("signals", s, 16000, lay=lays[i % 4], align=aligns[i % 4]))
    out.append(_case("signals", "noise", 16000, bank="slaney128", clamp=0.0))
    out.append(_case("signals", "silence", 9000, bank="slaney128", clamp=0.0, lay="fm"))
    out.append(_case("signals", "silence_tiny", 9000, clamp=0.0, align="mis"))
    out.append(_case("signals", "noise", 9000, clamp=1.0, lay="pad"))
    out.append(_case("signals", "int16", 9000, bank="slaney128", clamp=1.0, align="odd"))
    out.append(_case("signals", "mixture", 9000, bank="slaney128", win="rand"))
    # ---- bin probes: all 513 bins of every frame, directly
    for i, s in enumerate(("noise", "mixture", "tone_lanes", "chirp", "impulses", "tone_nyq", "tone_256")):
        for j in range(5):
            n = 5 * i + j
            out.append(_case("probes", s, (9000, 4865, 1023)[n % 3], bank=f"probe{j}", win=("hann", "rand", "hamming")[i % 3],
                             lay=lays[n % 4], align=aligns[(n + 1) % 4]))
    # ---- windows and banks
    for i, w in enumerate(("rand", "hamming")):
        for j, b in enumerate(("slaney80", "slaney128", "wide")):
            out.append(_case("windows", ("noise", "impulses", "chirp")[(i + j) % 3], 9000, win=w, bank=b,
                             lay=lays[(i + j) % 4], align=aligns[(i + 2 * j) % 4]))
    for i, b in enumerate(("slaney1", "slaney6", "slaney127", "wide")):
        for j, s in enumerate(("noise", "tone_half", "mixture")):
            out.append(_case("banks", s, (9000, 16000, 4864)[(i + j) % 3], bank=b, lay=lays[(i + j) % 4],
                             align=aligns[(i + 2 * j) % 4], win=("hann", "rand")[j % 2]))
    # ---- lengths: clip edges, the 4864-sample span and the 16-frame tile edge
    lengths = (513, 514, 767, 768, 1023, 1024, 1025, 4864, 4865, 3839, 3840, 4096, 7935, 8191, 8192)
    for i, n in enumerate(lengths):
        for j, b in enumerate(("slaney80", "slaney128")):
            out.append(_case("lengths", ("noise", "impulses", "tone_half")[(i + j) % 3], n, bank=b,
                             lay=lays[(i + j) % 4], align=aligns[(i + 3 * j) % 4]))
    # ---- every staging path with every store order, on both filterbank paths
    for b in ("slaney80", "slaney128"):
        for a in ("vec", "mis", "odd"):
            for k, lay in enumerate(lays):
                out.append(_case("paths", ("noise", "chirp", "mixture", "impulses")[k], 9000 + 257 * k, bank=b, lay=lay,
                                 align=a))
    # ---- ragged batches: each clip reflects at and counts frames to its own end; the last length exceeds L_max
    rag = (513, 1025, 4865, 16000, 9001, 20000)
    for i, (b, s) in enumerate((("slaney80", "impulses"), ("slaney128", "noise"), ("probe2", "chirp"),
                                ("slaney6", "mixture"), ("slaney80", "int16"))):
        out.append(_case("ragged", s, 16003, lens=rag[i:] + rag[:i], bank=b, lay=lays[i % 4], align=aligns[(i + 1) % 4]))
    return out


CASES = _cases()


def case_id(c):
    lens = "-rag" + "_".join(map(str, c["lens"])) if c["lens"] else ""
    return f"{c['block']}-{c['sig']}-L{c['L']}{lens}-{c['win']}-{c['bank']}-c{c['clamp']:g}-{c['lay']}-{c['align']}"


CASE_BY_ID = {case_id(c): c for c in CASES}


@functools.lru_cache(maxsize=None)
def inputs(cid):
    """(wav (B, L) fp32 with garbage past each clip's length, lens or None)"""
    c = CASE_BY_ID[cid]
    rng = np.random.default_rng(zlib.crc32(cid.encode()))
    lens = c["lens"]
    B = len(lens) if lens else 2
    wav = rng.uniform(-1e3, 1e3, (B, c["L"]))
    for b in range(B):
        n = min(lens[b], c["L"]) if lens else c["L"]
        wav[b, :n] = signal(c["sig"], n, rng)
    return wav.astype(np.float32), lens


@functools.lru_cache(maxsize=None)
def case_reference(cid):
    c = CASE_BY_ID[cid]
    wav, lens = inputs(cid)
    return RM.reference(wav, lens, window(c["win"]), bank(c["bank"])[0], c["clamp"])


# ------------------------------------------------------------------------------------------ the kernel's branches
def out_strides(lay, M, F):
    """(sb, sm, sf) of each output layout; the padded ones leave gaps that must keep the sentinel"""
    return dict(mm=(M * F, F, 1), fm=(F * M, 1, M), pad=(M * (F + 3) + 5, F + 3, 1),
                padfm=(F * (M + 2) + 7, 1, M + 2))[lay]


def paths(c):
    """what mel_kernel branches on, per CTA: (staged, staging, store order) and the case-wide axes"""
    fb, fb_w, fb_off, _ = bank(c["bank"])
    M = fb.shape[1]
    staged = int(fb_off[(M + 3) // 4]) <= FBW
    vec_ok = c["align"] == "vec"                        # 16-byte aligned base and a row stride divisible by 4
    sb, sm, sf = out_strides(c["lay"], M, 1 + c["L"] // HOP)
    order = "frames-fast" if sf <= sm else "mels-fast"
    ctas, tails, both_ends = set(), set(), False
    for n in (c["lens"] or (c["L"],)):
        Lb = min(n, c["L"])
        F = 1 + Lb // HOP
        tails.add(F % FPB)
        both_ends |= any(f * HOP - 512 < 0 and f * HOP + 511 >= Lb for f in range(F))
        for f0 in range(0, F, FPB):
            g0 = f0 * HOP - 512
            inside = g0 >= 0 and g0 + SPAN <= Lb
            ctas.add((staged, "vector" if vec_ok and inside else "scalar-interior" if inside else "scalar-edge", order))
    return dict(staged=staged, ctas=ctas, tails=tails, both_ends=both_ends, partial_groups=M % 4 != 0,
                ragged=c["lens"] is not None)


# ------------------------------------------------------------------------------------------ wrong front ends
def _bf16(a):
    i = np.asarray(a, np.float32).view(np.uint32).astype(np.uint64)
    i = (i + 0x7FFF + ((i >> 16) & 1)) & 0xFFFF0000
    return i.astype(np.uint32).view(np.float32).astype(np.float64)


def _fft_bf16_twiddles(x):
    n = x.shape[-1]
    if n == 1:
        return x.astype(np.complex128)
    e, o = _fft_bf16_twiddles(x[..., 0::2]), _fft_bf16_twiddles(x[..., 1::2])
    t = np.exp(-2j * np.pi * np.arange(n // 2) / n)
    t = (_bf16(t.real) + 1j * _bf16(t.imag)) * o
    return np.concatenate([e + t, e - t], -1)


def _shift_bank(fb):
    s = np.zeros_like(fb)
    s[1:] = fb[:-1]
    return s


WRONG = {
    "symmetric padding": lambda w, fb: dict(window=w, fb=fb, pad="symmetric"),
    "window reversed": lambda w, fb: dict(window=w[::-1].copy(), fb=fb),
    "bins k and 512-k swapped": lambda w, fb: dict(window=w, fb=fb, rfft=lambda a, axis: np.fft.rfft(a, axis=axis)[..., ::-1]),
    "bf16 twiddles": lambda w, fb: dict(window=w, fb=fb, rfft=lambda a, axis: _fft_bf16_twiddles(a)[..., :513]),
    "bank read one bin late": lambda w, fb: dict(window=w, fb=_shift_bank(fb)),
}


def _fp32_restatement(wav, lens, win, fb, clamp):
    return RM.spectrogram(wav, lens, win, fb, clamp, dtype=np.float32, rfft=lambda a, axis: scipy.fft.rfft(a, axis=axis))


# ------------------------------------------------------------------------------------------ CPU
def test_grouped_banks_unpack_to_the_dense_banks():
    for name in sorted({c["bank"] for c in CASES} | {"mixed128"} | {f"probe{j}" for j in range(5)}):
        fb, w, off, st = bank(name)
        assert np.array_equal(RM.unpack_grouped(w, off, st, fb.shape[1]), fb), name
    # the two filterbank paths: Slaney 80 is staged, Slaney 128 is not; mixed128's first 20 groups are Slaney 80's
    assert int(bank("slaney80")[2][-1]) == 1344 <= FBW < int(bank("slaney128")[2][-1]) == 1584
    s80, mix = bank("slaney80"), bank("mixed128")
    assert np.array_equal(mix[1][:1344], s80[1]) and np.array_equal(mix[2][:21], s80[2])
    assert np.array_equal(mix[3][:80], s80[3]) and int(mix[2][-1]) > FBW


def test_reference_admits_fp32_front_ends():
    """An fp32 restatement (scipy's fp32 FFT) on every case, and the fp32 torch.stft oracle on every case it can express
    (periodic Hann, a Slaney bank), stay within the bar."""
    from oracle import ref_megatts2 as R
    worst = {"fp32 restatement": 0.0, "torch.stft oracle": 0.0}
    for c in CASES:
        cid = case_id(c)
        wav, lens = inputs(cid)
        fb = bank(c["bank"])[0]
        ref, bar = case_reference(cid)
        r = RM.excess(_fp32_restatement(wav, lens, window(c["win"]), fb, c["clamp"]), ref, bar).max()
        assert r <= 1, (cid, "fp32 restatement", r)
        worst["fp32 restatement"] = max(worst["fp32 restatement"], r)
        if c["win"] == "hann" and c["bank"].startswith("slaney"):
            out = np.full_like(ref, np.nan)
            for b in range(wav.shape[0]):
                n = min(lens[b], c["L"]) if lens else c["L"]
                o = R.mel_spectrogram(torch.from_numpy(wav[b, :n])[None], n_mels=fb.shape[1], clamp=c["clamp"])[0]
                out[b, :, :o.shape[1]] = o.numpy()
            r = RM.excess(out, ref, bar).max()
            assert r <= 1, (cid, "torch.stft", r)
            worst["torch.stft oracle"] = max(worst["torch.stft oracle"], r)
    print(worst)


TIGHT = 1e-2


def test_bar_rejects_plausible_wrong_front_ends():
    """Each wrong variant misses the bar by at least 4x somewhere in every case it visibly changes.  Visible: it moves an
    element whose bar is at most 1 % by more than 1 % (log domain), or turns an infinity finite or back.  Elements with a
    wider bar are bands far below their frame's energy, where fp32 itself cannot tell these variants apart; and some
    variants are near no-ops on some inputs (reversing a symmetric window shifts it by one sample; swapping bins k and
    512 - k leaves a tone at bin 256 alone)."""
    least = {name: (math.inf, None, 0) for name in WRONG}
    for c in CASES:
        cid = case_id(c)
        wav, lens = inputs(cid)
        ref, bar = case_reference(cid)
        tight = ~np.isnan(ref) & (bar <= TIGHT)
        w, fb = window(c["win"]), bank(c["bank"])[0]
        for name, make in WRONG.items():
            kw = make(w, fb)
            out = RM.spectrogram(wav, lens, kw.pop("window"), kw.pop("fb"), c["clamp"], **kw)
            r = RM.excess(out, ref, bar)[tight]
            with np.errstate(invalid="ignore"):
                moved = np.nan_to_num(np.abs(out - ref)[tight], nan=0.0, posinf=0.0)
            if moved.max(initial=0) <= TIGHT and np.isfinite(r).all():
                continue
            assert r.max() >= 4, (cid, name, r.max())
            least[name] = min(least[name][:2], (r.max(), cid)) + (least[name][2] + 1,)
    for name, (r, cid, n) in least.items():
        assert n >= 50, (name, n)
        print(f"{name}: changes {n} of {len(CASES)} cases, at least {r:.1f}x the bar (smallest at {cid})")


def test_case_table_reaches_every_path():
    assert len(CASE_BY_ID) == len(CASES)
    assert (HOP, FPB, SPAN) == (256, 16, 1024 + 15 * 256)
    seen, tails = set(), {True: set(), False: set()}
    for c in CASES:
        p = paths(c)
        seen |= p["ctas"]
        s = p["staged"]
        tails[s] |= p["tails"]
        seen |= {(s, "ragged", p["ragged"]), (s, "n_mels % 4", p["partial_groups"]), (s, "both ends", p["both_ends"])}
        seen.add(("window", c["win"], s))
    for s in (True, False):
        for st in ("vector", "scalar-interior", "scalar-edge"):
            for order in ("frames-fast", "mels-fast"):
                assert (s, st, order) in seen, (s, st, order)
        for axis in ("ragged", "n_mels % 4", "both ends"):
            assert (s, axis, True) in seen and (s, axis, False) in seen, (s, axis)
        assert {0, 1, FPB - 1} <= tails[s], (s, tails[s])
        for w in ("hann", "rand", "hamming"):
            assert ("window", w, s) in seen, (w, s)
    assert {c["sig"] for c in CASES} == set(SIGNALS)
    assert {c["clamp"] for c in CASES} == {1e-5, 0.0, 1.0}
    assert {c["lay"] for c in CASES} == {"mm", "fm", "pad", "padfm"}
    lengths = {min(n, c["L"]) for c in CASES for n in (c["lens"] or (c["L"],))}
    assert {513, 514, 767, 768, 1023, 1024, 1025, 4864, 4865} <= lengths
    assert any(c["lens"] and max(c["lens"]) > c["L"] for c in CASES)
    # bin probes: each signal probed covers bins 0..512 once, at every start alignment
    for s in {c["sig"] for c in CASES if c["block"] == "probes"}:
        bins = sorted(k for c in CASES if c["block"] == "probes" and c["sig"] == s
                      for k in np.nonzero(bank(c["bank"])[0])[0])
        assert bins == list(range(513)), s


# ------------------------------------------------------------------------------------------ GPU
class Tables:
    def __init__(self, win, bank_name):
        fb, fb_w, fb_off, fb_start = bank(bank_name)
        self.M = fb.shape[1]
        self.window = torch.from_numpy(window(win)).to(DEV)
        self.fb_w = torch.from_numpy(fb_w).to(DEV)
        self.fb_off = torch.from_numpy(fb_off).to(DEV)
        self.fb_start = torch.from_numpy(fb_start).to(DEV)


def wav_buffer(wav, align):
    """the clips on the device with the row stride and base alignment `align` asks for: (buffer, offset, row stride)"""
    B, n = wav.shape
    sb = (n + 3) // 4 * 4 + (align == "odd")
    off = int(align == "mis")
    host = torch.full((off + B * sb + 4,), 1e3)
    torch.as_strided(host, (B, n), (sb, 1), off).copy_(torch.from_numpy(wav))
    return host.to(DEV), off, sb


def launch(wav, lens, tabs, clamp, lay="mm", align="vec", L=None, n_mels=None, window_ptr=None,
           fb_w_ptr=None, check=True):
    """one call of the C entry point (ragged when lens is given) -> (out (B, n_mels, F) fp32 on the host, the whole
    output buffer, its strides, the return code)"""
    from megatts2_b200 import ops
    B, Lw = wav.shape
    L = Lw if L is None else L
    M = tabs.M if n_mels is None else n_mels
    F = 1 + L // HOP
    buf, off, wsb = wav_buffer(wav, align)
    sb, sm, sf = out_strides(lay, max(M, 1), F)
    size = (B - 1) * sb + (max(M, 1) - 1) * sm + (F - 1) * sf + 1 + 16
    out = torch.full((size,), SENTINEL, device=DEV)
    wp = buf.data_ptr() + 4 * off
    tab = (window_ptr or tabs.window.data_ptr(), fb_w_ptr or tabs.fb_w.data_ptr(), tabs.fb_off.data_ptr(),
           tabs.fb_start.data_ptr())
    if lens is None:
        rc = LIB.lib().mtts_mel_spectrogram_f32(wp, wsb, B, L, *tab, M, clamp, out.data_ptr(), sb, sm, sf, ops._stream())
    else:
        ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
        rc = LIB.lib().mtts_mel_spectrogram_ragged_f32(wp, wsb, B, L, ld.data_ptr(), *tab, M, clamp, out.data_ptr(), sb, sm,
                                                      sf, ops._stream())
    torch.cuda.synchronize()
    if check:
        LIB.check(rc)
    out = out.cpu()
    view = torch.as_strided(out, (B, max(M, 1), F), (sb, sm, sf)).numpy().copy()
    return view, out, (sb, sm, sf), rc


def written_mask(size, B, M, F_of, strides):
    w = torch.zeros(size, dtype=torch.bool)
    v = torch.as_strided(w, (B, M, max(F_of)), strides)
    for b in range(B):
        v[b, :, :F_of[b]] = True
    return w


def frame_counts(L, lens, B):
    return [1 + (min(n, L) if lens else L) // HOP for n in (lens or (L,) * B)]


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_mel_vs_fp64(c):
    cid = case_id(c)
    wav, lens = inputs(cid)
    B = wav.shape[0]
    tabs = Tables(c["win"], c["bank"])
    out, buf, strides, _ = launch(wav, lens, tabs, c["clamp"], c["lay"], c["align"])
    again, _, _, _ = launch(wav, lens, tabs, c["clamp"], c["lay"], c["align"])
    assert np.array_equal(out.view(np.int32), again.view(np.int32)), "a repeat launch differs"
    # frames a clip does not have, and the gaps of a padded layout, keep the sentinel
    F_of = frame_counts(c["L"], lens, B)
    keep = ~written_mask(buf.numel(), B, tabs.M, F_of, strides)
    assert bool((buf[keep] == SENTINEL).all()), "the kernel wrote outside the clips' frames"
    ref, bar = case_reference(cid)
    r = RM.excess(out, ref, bar)
    ratio = float(r.max())
    err = np.abs(out.astype(np.float64) - ref)[~np.isnan(ref) & np.isfinite(ref) & np.isfinite(out)]
    print(f"{cid}: staged {paths(c)['staged']}  error / bar {ratio:.3f}")
    helpers.record("mel_oracle", dict(case=cid, cls=c["block"], staged=paths(c)["staged"], err_to_bound=ratio,
                                      max_err=float(err.max(initial=0))))
    if not ratio <= 1:
        i = np.unravel_index(int(np.argmax(r)), r.shape)
        pytest.fail(f"error is {ratio:.2f}x the bar at (b, m, f) = {i}: {out[i]!r} against {ref[i]!r}, bar {bar[i]:.3e}")


def _noise(B, n, seed):
    return np.random.default_rng(seed).uniform(-1, 1, (B, n)).astype(np.float32)


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


@gpu
def test_clip_alone_equals_plain_and_ragged_batch():
    wav = _noise(3, 9000, 1)
    for name in ("slaney80", "slaney128"):
        tabs = Tables("hann", name)
        batch = launch(wav, None, tabs, 1e-5)[0]
        for b in range(3):
            assert np.array_equal(_bits(launch(wav[b:b + 1], None, tabs, 1e-5)[0][0]), _bits(batch[b])), (name, b)
        lens = (513, 9000, 5000)
        rag = launch(wav, lens, tabs, 1e-5)[0]
        assert np.array_equal(_bits(rag[1]), _bits(batch[1])), name
        alone = launch(np.ascontiguousarray(wav[2:3, :5000]), None, tabs, 1e-5)[0][0]
        assert np.array_equal(_bits(rag[2, :, :alone.shape[1]]), _bits(alone)), name
        alone = launch(np.ascontiguousarray(wav[0:1, :513]), None, tabs, 1e-5)[0][0]
        assert np.array_equal(_bits(rag[0, :, :alone.shape[1]]), _bits(alone)), name


@gpu
def test_vector_and_scalar_staging_agree():
    wav = _noise(2, 16000, 2)
    for name in ("slaney80", "slaney128"):
        tabs = Tables("rand", name)
        vec = launch(wav, None, tabs, 1e-5, align="vec")[0]
        for a in ("mis", "odd"):
            assert np.array_equal(_bits(launch(wav, None, tabs, 1e-5, align=a)[0]), _bits(vec)), (name, a)


@gpu
def test_staged_and_global_filterbank_agree():
    wav = _noise(2, 9000, 3)
    s80 = launch(wav, None, Tables("hann", "slaney80"), 1e-5)[0]
    mix = launch(wav, None, Tables("hann", "mixed128"), 1e-5)[0]
    assert np.array_equal(_bits(mix[:, :80]), _bits(s80))


@gpu
def test_output_layouts_agree():
    wav = _noise(2, 5000, 4)
    for name in ("slaney80", "slaney127"):
        tabs = Tables("hann", name)
        mm = launch(wav, None, tabs, 1e-5, lay="mm")[0]
        for lay in ("fm", "pad", "padfm"):
            assert np.array_equal(_bits(launch(wav, None, tabs, 1e-5, lay=lay)[0]), _bits(mm)), (name, lay)


@gpu
@pytest.mark.timeout(300)
def test_batch_fold_past_65535():
    """B = 65539 runs as two launches; the second's clips, lengths and outputs are offset by 65535"""
    B, n = 65539, 516
    wav = _noise(B, n, 5)
    lens = [513 + (b * 7) % 4 for b in range(B)]
    tabs = Tables("hann", "slaney80")
    plain = launch(wav, None, tabs, 1e-5, L=513)[0]
    rag = launch(wav, lens, tabs, 1e-5)[0]
    for b in range(B - 5, B):
        one = launch(wav[b:b + 1], None, tabs, 1e-5, L=513)[0][0]
        assert np.array_equal(_bits(plain[b]), _bits(one)), b
        one = launch(np.ascontiguousarray(wav[b:b + 1, :lens[b]]), None, tabs, 1e-5)[0][0]
        assert np.array_equal(_bits(rag[b]), _bits(one)), b
        ref, bar = RM.reference(wav[b:b + 1, :lens[b]], None, window("hann"), bank("slaney80")[0], 1e-5)
        assert RM.excess(one[None], ref, bar).max() <= 1, b


@gpu
def test_refusals_launch_nothing():
    from megatts2_b200 import ops
    wav = _noise(2, 2000, 6)
    tabs = Tables("hann", "slaney80")
    w_off = torch.zeros(1024 + 4, device=DEV)
    w_off[1:1025] = tabs.window
    fb_off = torch.zeros(tabs.fb_w.numel() + 4, device=DEV)
    fb_off[1:1 + tabs.fb_w.numel()] = tabs.fb_w
    bad = [dict(L=512), dict(ragged_L=512), dict(n_mels=0), dict(n_mels=129),
           dict(window_ptr=w_off.data_ptr() + 4), dict(fb_w_ptr=fb_off.data_ptr() + 4)]
    for kw in bad:
        n0 = ops.launch_count()
        if "ragged_L" in kw:
            _, buf, _, rc = launch(np.ascontiguousarray(wav[:, :512]), (512, 512), tabs, 1e-5, check=False)
        else:
            _, buf, _, rc = launch(wav, None, tabs, 1e-5, check=False, **kw)
        assert rc != 0, kw
        assert ops.launch_count() == n0, kw
        assert bool((buf == SENTINEL).all()), kw
