"""CPU: long-form synthesis's host side - every validation error of Megatts.synthesize_passage / _stream and every
rejected argument, the window / key / layout rules against the restatement (tests/ref_passage.py), the entries a passage
enqueues (the library replaced by a recorder and each sentence's synthesis by a stand-in), the C argument checks and the
ctypes mirror of mtts_copy_row_segments."""
import ctypes as C
import functools
import os
import random
import re

import pytest
import torch

import ref_passage as RP
from conftest import ROOT
from megatts2_b200 import _lib as L
from megatts2_b200 import graphs, ops
from megatts2_b200 import passage as PS
from megatts2_b200.models.megatts2 import Megatts, PLMContext
from megatts2_b200.modules.mrte import MRTE
from megatts2_b200.sampling import Sampling

B, NB, TC = 2, 80, 512
COPY = "mtts_copy_row_segments"


class Recorder:
    """Stands in for the library: records the entry names (and the integer arguments of mtts_copy_row_segments)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return functools.partial(self._call, name)

    def _call(self, name, *args):
        assert len(args) == len(L.SIGNATURES[name][1]), name
        if name == COPY:
            ints = (C.c_int32, C.c_int64, C.c_uint32)
            self.calls.append((name, tuple(a for a, t in zip(args, L.SIGNATURES[name][1]) if t in ints)))
        else:
            self.calls.append(name)
        if name.endswith("_workspace_bytes") or name == "mtts_linear_tc_scratch_bytes":
            return 4096
        if name == "mtts_convnet_double_out_len":
            return (args[1] - 1) // 16 + 1
        return 0


@pytest.fixture
def lib(monkeypatch):
    rec = Recorder()
    monkeypatch.setattr(L, "lib", lambda: rec)
    monkeypatch.setattr(ops, "_dev", lambda t, dtype=torch.float32, name="tensor": _cpu_dev(t, dtype, name))
    monkeypatch.setattr(ops, "workspace", lambda nbytes, device: torch.empty(int(nbytes) + 256, dtype=torch.uint8))
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0x5EA))
    monkeypatch.setattr(ops, "tc_overflow_bind", lambda device: None)
    monkeypatch.setattr(graphs, "_enabled", True)
    return rec


def _cpu_dev(t, dtype, name):
    if not isinstance(t, torch.Tensor) or t.dtype != dtype:
        raise L.MttsError(f"{name}: expected a {dtype} tensor")
    return t


def _mrte():
    return MRTE(hidden_size=32, content_ff_dim=64, content_n_layers=1, mel_n_layer=1, mel_n_stack=1,
                mel_n_block=1).eval()


class _Voc:
    cfg = dict(inference_padding=5)

    def __init__(self):
        self.calls = []

    def receptive_field(self):
        return 14

    def decode_batch_cl(self, mel):
        self.calls.append(tuple(mel.shape))
        return torch.zeros(mel.shape[0], 1, 256 * (mel.shape[1] + 10))


def _tts(mrte=None):
    tts = Megatts.__new__(Megatts)
    torch.nn.Module.__init__(tts)
    tts.generator = type("G", (), {"mrte": mrte if mrte is not None else _mrte()})()
    tts.plm = type("P", (), {"vq_bins": 1024, "tc_latent_dim": TC})()
    voc = _Voc()
    tts.hifi_gan = type("H", (), {"generator": voc, "decode_batch_cl": voc.decode_batch_cl})()
    return tts


def _sents(Tps=(3, 5, 4)):
    return [torch.randint(0, 320, (B, t)) for t in Tps]


def _mel(T=40):
    return torch.randn(B, T, NB)


def _ctx(Bc, P=3):
    c = PLMContext.__new__(PLMContext)
    c.tc8, c.codes, c.max_code = torch.rand(Bc, P, TC), torch.randint(0, 1024, (Bc, P)), 1023
    return c


# ------------------------------------------------------------------------------ validation
BAD = [
    (dict(sentences=[]), "sentences must be a non-empty list"),
    (dict(sentences="tensor"), "sentences must be a non-empty list"),
    (dict(sentences=["f32"]), r"sentences\[0\]: expected a \(B, Tp >= 1\) int64"),
    (dict(sentences=["ok", "rows"]), r"sentences\[1\]: \(3, 4\) on cpu, expected B = 2"),
    (dict(sentences=["ok", "empty"]), r"sentences\[1\]: expected a \(B, Tp >= 1\)"),
    (dict(mels="short"), r"mels: expected a \(2, Tm >= 1, 80\) float32 tensor"),
    (dict(mels="bins"), r"mels: expected a \(2, Tm >= 1, 80\)"),
    (dict(context_rows=-1), "context_rows must be an int >= 0"),
    (dict(context_rows=True), "context_rows must be an int >= 0"),
    (dict(context_rows=1.5), "context_rows must be an int >= 0"),
    (dict(pause_frames=-2), "pause_frames must be >= 0"),
    (dict(pause_frames=[[1, 2]]), r"pause_frames: shape \(1, 2\), expected an int or \(2, 2\)"),
    (dict(pause_frames=[[1, 2], [3, -1]]), r"pause_frames\[1, 1\] = -1: the pause after sentence 1 of row 1"),
    (dict(pause_frames=[[1.0, 2.0], [3.0, 1.0]]), "pause_frames: expected integers"),
    (dict(plm_context="B3"), r"plm_context: Bc = 3, expected 1 or B = 2"),
    (dict(plm_context="dim"), r"plm_context: latents \(Bc, P, 512\)"),
    (dict(plm_context="code"), r"plm_context: codes must be in \[0, 1024\)"),
    (dict(forced_durations="tensor"), "forced_durations: expected a list of 3"),
    (dict(forced_durations="two"), "forced_durations: expected a list of 3"),
    (dict(forced_durations="shape"), r"forced_durations\[1\]: shape \(2, 4\), expected \(2, 5\)"),
    (dict(forced_durations="neg"), r"forced_durations\[2\]\[1, 3\] = -1: durations must be >= 0"),
    (dict(forced_durations="ok", duration_scale=1.2), "do not combine with duration_scale"),
    (dict(duration_scale=0.0), "duration_scale: every value must be finite and > 0"),
    (dict(duration_scale=[1.0, 1.0, 1.0]), r"duration_scale: shape \(3,\)"),
    (dict(duration_scale="per_phone"), r"duration_scale: shape \(2, 3\), expected \(\) or \(2,\)"),
    (dict(sampling="greedy"), "sampling must be a megatts2_b200.sampling.Sampling"),
    (dict(sampling=Sampling(seed=1), keys=[1, 2, 3]), r"keys: expected shape \(2,\)"),
]


def _resolve(kw):
    kw = dict(kw)
    named = {"ok": torch.zeros(B, 3, dtype=torch.int64), "f32": torch.zeros(B, 3), "rows": torch.zeros(3, 4, dtype=torch.int64),
             "empty": torch.zeros(B, 0, dtype=torch.int64)}
    if kw.get("sentences") == "tensor":
        kw["sentences"] = torch.zeros(B, 3, dtype=torch.int64)
    elif "sentences" in kw:
        kw["sentences"] = [named[s] for s in kw["sentences"]]
    kw["mels"] = {"short": torch.zeros(1, 40, NB), "bins": torch.zeros(B, 40, 81)}.get(kw.get("mels"), _mel())
    if isinstance(kw.get("plm_context"), str):
        c = _ctx(3 if kw["plm_context"] == "B3" else B)
        if kw["plm_context"] == "dim":
            c.tc8 = torch.zeros(B, 3, 16)
        if kw["plm_context"] == "code":
            c.max_code = 1024
        kw["plm_context"] = c
    sents = kw.get("sentences") if "sentences" in kw else _sents()
    fd = kw.get("forced_durations")
    if isinstance(fd, str):
        good = [torch.full(tuple(s.shape), 2, dtype=torch.int32) for s in _sents()]
        kw["forced_durations"] = {"tensor": good[0], "two": good[:2], "ok": good,
                                  "shape": [good[0], good[2], good[2]],
                                  "neg": good[:2] + [good[2].clone().index_put_((torch.tensor(1), torch.tensor(3)),
                                                                                 torch.tensor(-1, dtype=torch.int32))]}[fd]
    if kw.get("duration_scale") == "per_phone":
        kw["duration_scale"] = torch.ones(B, 3)
    return sents, kw


@pytest.mark.parametrize("kw, match", BAD)
@pytest.mark.parametrize("entry", ["synthesize_passage", "synthesize_passage_stream"])
def test_rejects_bad_arguments(lib, kw, match, entry):
    sents, kw = _resolve(kw)
    kw.pop("sentences", None)
    mels = kw.pop("mels")
    with pytest.raises(L.MttsError, match=match):
        getattr(_tts(), entry)(sents, mels, **kw)            # the stream raises before its first next
    assert lib.calls == []


@pytest.mark.parametrize("name", sorted(PS.REJECTED))
@pytest.mark.parametrize("entry", ["synthesize_passage", "synthesize_passage_stream"])
def test_rejects_synthesize_arguments_by_name(lib, name, entry):
    with pytest.raises(L.MttsError, match=f"synthesize_passage does not take {name}: "):
        getattr(_tts(), entry)(_sents(), _mel(), **{name: None})
    with pytest.raises(TypeError, match="unexpected keyword"):
        getattr(_tts(), entry)(_sents(), _mel(), no_such_argument=1)
    assert lib.calls == []


# ------------------------------------------------------------------------------ the rules against the restatement
def test_keys_wrap_in_int64():
    for k in (0, 5, -1, 2 ** 63 - 1, -2 ** 63, 2 ** 62):
        for i in range(4):
            assert PS.sentence_keys([k], i) == [RP.key(k, i)]
    assert PS.sentence_keys([2 ** 63 - 1], 1) == [-2 ** 63 + 2 ** 32 - 1]


def _simulate(P0, totals, context_rows):
    """The planner's (window P, kept rows per row) sentence by sentence, with the rows identified as in ref_passage."""
    Bn = len(totals[0])
    kept = [[("ctx", j) for j in range(P0)] for _ in range(Bn)]
    count, H, got = [P0] * Bn, [P0] * Bn, []
    for s, t in enumerate(totals):
        P = PS.window_rows(H, context_rows)
        got.append((P, [k[len(k) - P:] for k in kept] if P else None))
        n = PS.codes_rows(t)
        keep, o, m = PS.history_update(count, n, context_rows)
        kept = [k[len(k) - ob:] if ob else [] for k, ob in zip(kept, o)]
        kept = [k + [(s, j) for j in range(nb - mb, nb)] for k, nb, mb in zip(kept, n, m)]
        assert [len(k) for k in kept] == keep
        count, H = keep, [h + nb for h, nb in zip(H, n)]
    return got


@pytest.mark.parametrize("seed", range(40))
def test_window_rule_against_the_restatement(seed):
    r = random.Random(seed)
    Bn, S_ = r.randint(1, 5), r.randint(1, 6)
    P0 = r.choice([0, 0, 1, 7, 40])
    context_rows = r.choice([0, 1, 5, 16, 128])
    totals = [[r.choice([0, 1, 7, 8, 9, 30, 100]) for _ in range(Bn)] for _ in range(S_)]
    got = _simulate(P0, totals, context_rows)
    for i in range(S_):
        P, rows = RP.window(P0, totals[:i], context_rows) if i else (min(context_rows, P0), None)
        assert got[i][0] == P, (i, got[i][0], P)
        if i and P:
            assert got[i][1] == rows, i


def test_window_edge_cases():
    # a row whose history is shorter than context_rows binds every row (min_b H_b)
    assert _simulate(0, [[8, 800], [8, 8]], 128)[1][0] == 1
    assert _simulate(0, [[80, 800], [8, 8]], 128)[1][0] == 10
    # the initial context alone, then capped by context_rows
    assert _simulate(200, [[8, 8]], 128)[0][0] == 128
    # zero-frame sentences add no rows
    assert _simulate(0, [[0, 0], [8, 8]], 128)[1][0] == 0
    assert _simulate(3, [[0, 16], [8, 8]], 128)[1] == (3, [[("ctx", 0), ("ctx", 1), ("ctx", 2)],
                                                           [("ctx", 2), (0, 0), (0, 1)]])


@pytest.mark.parametrize("seed", range(20))
def test_layout_against_the_restatement(seed):
    r = random.Random(seed)
    Bn, S_ = r.randint(1, 4), r.randint(1, 5)
    totals = [[r.randint(0, 40) for _ in range(Bn)] for _ in range(S_)]
    pauses = [[r.randint(0, 30) for _ in range(S_ - 1)] for _ in range(Bn)]
    offs, F = PS.frame_offsets(totals, pauses)
    frames, want = RP.layout(totals, pauses)
    assert offs == want and F == [len(f) for f in frames]
    pad = 5
    for b in range(Bn):                                  # the chunks tile the padded waveform
        pos = 0
        for i in range(S_):
            p0, p1 = PS.chunk_bounds(offs, totals, F, i, pad)[b]
            assert p0 == pos
            pos = p1
        assert pos == F[b] + 2 * pad


# ------------------------------------------------------------------------------ dispatch
def _fake_synthesize(log, totals_by_sentence):
    def fake(self, phone, mels, forced, causal, prompt, overlap, sampling, keys, pm, pw, dw, ctx, control,
             mel_context=None, mel_only=False):
        i = len(log)
        log.append(dict(ctx=ctx, keys=keys, mel_context=mel_context, mel_only=mel_only, graphs=graphs.enabled(),
                        forced=forced, control=control))
        totals = totals_by_sentence[i]
        T8 = -(-max(totals) // 8)
        return dict(tc8=torch.rand(B, T8, TC), p_codes=torch.randint(0, 1024, (B, T8)), dt=torch.ones(B, 3),
                    mel=torch.rand(B, max(totals), NB), totals=totals)
    return fake


def test_dispatch_one_encoder_pass_and_one_copy_per_join(lib, monkeypatch):
    log, totals = [], [[20, 12], [9, 30], [16, 16]]
    monkeypatch.setattr(Megatts, "_synthesize", _fake_synthesize(log, totals))
    tts = _tts()
    ctx = _ctx(1, P=3)
    out = tts.synthesize_passage(_sents(), _mel(), pause_frames=[[2, 0], [1, 4]], plm_context=ctx, context_rows=4,
                                 sampling=Sampling(seed=3), keys=[7, -1], return_intermediates=True, check_range=False)
    assert sum(c == "mtts_convnet_double_forward_f32" for c in lib.calls) == 1        # the prompt, once per passage
    assert all(e["mel_only"] and not e["graphs"] for e in log)
    assert all(e["mel_context"] is log[0]["mel_context"] for e in log)
    assert [e["keys"].tolist() for e in log] == [[RP.key(7, i), RP.key(-1, i)] for i in range(3)]
    assert out["context_rows_used"].tolist() == [3, 4, 4]
    assert [e["ctx"].P for e in log] == [3, 4, 4] and all(e["ctx"].tc8.shape[0] == B for e in log)
    copies = [c[1] for c in lib.calls if not isinstance(c, str)]
    assert all(c == COPY for c in lib.calls if isinstance(c, str) and "copy_row" in c)
    f4, i8 = 4 * TC, 8
    # (src_sb, src_st, src_rows, dst_sb, dst_st, dst_rows, row_bytes, B, n_max, fill_word)
    want = [
        (0, f4, 3, 3 * f4, f4, 3, f4, B, 3, 0), (0, i8, 3, 3 * i8, i8, 3, i8, B, 3, 0),      # W_0 from the Bc = 1 context
        # after sentence 0 (3 and 2 new rows) each row keeps 4: the last 1 / 2 context rows, then the new rows
        (0, f4, 3, 4 * f4, f4, 4, f4, B, 2, 0), (0, i8, 3, 4 * i8, i8, 4, i8, B, 2, 0),
        (3 * f4, f4, 3, 4 * f4, f4, 4, f4, B, 3, 0), (3 * i8, i8, 3, 4 * i8, i8, 4, i8, B, 3, 0),
    ]
    assert copies[:6] == want
    mel_copies = [c for c in copies if c[6] == NB * 4]
    assert len(mel_copies) == 3 + 2                                              # 3 sentences, 2 pause fills
    fills = [c for c in mel_copies if c[2] == 0]
    word = int(torch.tensor([PS.SILENCE]).view(torch.int32)) & 0xFFFFFFFF
    assert [c[9] for c in fills] == [word, word] and [c[8] for c in fills] == [2, 4]
    # per sentence after the first: a window (2 copies); per sentence but the last: a history update (2 or 4 copies)
    assert len(copies) - len(mel_copies) == 2 * 3 + 4 + 4
    offs, F = PS.frame_offsets(totals, [[2, 0], [1, 4]])
    assert out["frame_offsets"].tolist() == offs and out["wav_lens"] == [256 * (f + 10) for f in F]
    assert tts.hifi_gan.generator.calls == [(1, F[0], NB), (1, F[1], NB)]            # one vocode per passage length


def test_dispatch_without_context_makes_no_window_copies(lib, monkeypatch):
    log, totals = [], [[8, 8], [8, 8], [8, 8]]
    monkeypatch.setattr(Megatts, "_synthesize", _fake_synthesize(log, totals))
    tts = _tts()
    out = tts.synthesize_passage(_sents(), _mel(), context_rows=0, return_intermediates=True, check_range=False)
    assert [e["ctx"] for e in log] == [None] * 3 and [e["keys"] for e in log] == [None] * 3
    assert out["context_rows_used"].tolist() == [0, 0, 0]
    copies = [c[1] for c in lib.calls if not isinstance(c, str)]
    assert len(copies) == 3                                                       # the sentences' mel, no pauses
    assert tts.hifi_gan.generator.calls == [(B, 24, NB)]


def test_stream_dispatch_and_graph_state(lib, monkeypatch):
    log, totals = [], [[20, 12], [9, 30], [16, 16]]
    monkeypatch.setattr(Megatts, "_synthesize", _fake_synthesize(log, totals))
    tts = _tts()
    chunks = []
    for c in tts.synthesize_passage_stream(_sents(), _mel(), pause_frames=14, check_range=False):
        assert graphs.enabled()                                  # the caller's graphs stay on between chunks
        chunks.append((c["sentence"], len(log)))
    assert chunks == [(0, 1), (1, 2), (2, 3)]
    assert sum(c == "mtts_convnet_double_forward_f32" for c in lib.calls) == 1


# ------------------------------------------------------------------------------ C side
def _err():
    return L.lib().mtts_last_error().decode()


def test_c_side_rejects_bad_copy_arguments():
    """mtts_copy_row_segments checks every argument before it enqueues anything (so no device is needed to see the
    errors)."""
    lib_ = L.lib()
    d = C.c_void_p(256)                       # never dereferenced: every call below fails its checks first

    def call(src=C.c_void_p(1024), s_sb=4096, s_st=64, s_rows=8, dst=d, d_sb=4096, d_st=64, d_rows=8, rb=64,
             s_off=d, d_off=d, n=d, Bn=4, n_max=8):
        return lib_.mtts_copy_row_segments(src, s_sb, s_st, s_rows, dst, d_sb, d_st, d_rows, rb, s_off, d_off, n, Bn,
                                           n_max, 0, None)
    for kw in (dict(dst=None), dict(d_off=None), dict(n=None), dict(s_off=None)):
        assert call(**kw) == -1 and "null" in _err(), kw
    assert call(src=d) == -1 and "differ" in _err()
    for rb in (0, -4, 6):
        assert call(rb=rb) == -1 and "row_bytes" in _err(), rb
    for Bn in (-1, 65536):
        assert call(Bn=Bn) == -1 and "B must" in _err(), Bn
    assert call(n_max=-1) == -1 and "n_max" in _err()
    assert call(s_rows=-1) == -1 and "rows" in _err()
    for kw in (dict(s_st=32), dict(d_st=60), dict(s_sb=-4), dict(d_sb=2), dict(s_st=66)):
        assert call(**kw) == -1 and "strides" in _err(), kw
    assert call(d_sb=256) == -1 and "overlap" in _err()
    assert call(src=C.c_void_p(1026)) == -1 and "aligned" in _err()
    assert call(Bn=0) == 0 and call(n_max=0) == 0                       # nothing to do
    assert call(src=None, s_off=None, n_max=0) == 0                     # fill mode takes no src_off


def test_ctypes_signature_matches_the_header():
    src = open(os.path.join(ROOT, "include", "megatts2_b200.h")).read()
    m = re.search(r"\b" + COPY + r"\(([^)]*)\)", src)
    assert m
    args = [a.strip() for a in m.group(1).split(",") if a.strip()]
    types = L.SIGNATURES[COPY][1]
    assert len(types) == len(args) and L.SIGNATURES[COPY][0] is C.c_int
    want = {"int64_t": C.c_int64, "int32_t": C.c_int32, "uint32_t": C.c_uint32}
    for a, t in zip(args, types):
        base = a.rsplit(" ", 1)[0].replace("const ", "")
        assert t is (C.c_void_p if "*" in a else want[base]), a
    assert getattr(L.lib(), COPY) is not None
