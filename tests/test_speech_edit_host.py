"""CPU: speech editing's host side - the code-pin validator, the split of a pinned decode into runs of steps with a free
row, the pin rule of megatts2_b200/edit.py against its frame-by-frame restatement (tests/ref_speech_edit.py), every
validation error of Megatts.edit, the entries MegaPLM.infer calls with pins (the library replaced by a recorder), the C
argument checks and the ctypes mirror of the new entry."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import ref_speech_edit as RE
from conftest import ROOT
from megatts2_b200 import _lib as L
from megatts2_b200 import sampling as S
from megatts2_b200.edit import REJECTED, EditPlan
from megatts2_b200.models.megatts2 import Megatts, PLMContext
from test_plm_dispatch_host import M_PLM, P, SMP_STRUCT, WS_OK, Recorder, _latent, _plm, _smp, lib  # noqa: F401

V = 16                        # the recorder's PLM has vq_bins = 16


# ------------------------------------------------------------------------------ validator and runs
def test_pinned_codes_accepts_free_and_codes():
    p = S.pinned_codes([[-1, 0, 15], [3, -1, -1]], 2, 3, V)
    assert p.dtype == torch.int32 and p.tolist() == [[-1, 0, 15], [3, -1, -1]]
    assert S.pinned_codes(torch.full((2, 0), -1), 2, 0, V).shape == (2, 0)


@pytest.mark.parametrize("bad, where", [(V, "[1, 2]"), (V + 1, "[1, 2]"), (-2, "[1, 2]"), (-5, "[1, 2]"),
                                        (1 << 40, "[1, 2]")])
def test_pinned_codes_rejects_values(bad, where):
    p = torch.full((2, 3), -1, dtype=torch.int64)
    p[1, 2] = bad
    with pytest.raises(L.MttsError, match=re.escape(f"pinned codes{where} = {bad}")):
        S.pinned_codes(p, 2, 3, V)


def test_pinned_codes_rejects_shapes_and_types():
    for bad in (torch.zeros(2, 4, dtype=torch.int64), torch.zeros(3, 3, dtype=torch.int64), torch.zeros(2, 3)):
        with pytest.raises(L.MttsError, match="pinned codes"):
            S.pinned_codes(bad, 2, 3, V)


def test_runs():
    free = torch.full((3, 7), -1, dtype=torch.int32)
    assert S.pinned_runs(free) == ((0, 7),)
    assert S.pinned_runs(torch.zeros(3, 7, dtype=torch.int32)) == ()
    p = torch.zeros(3, 10, dtype=torch.int32)
    p[0, 2] = -1                                  # one free row is enough to run the step
    p[2, 3:5] = -1
    p[1, 9] = -1
    assert S.pinned_runs(p) == ((2, 5), (9, 10))
    p[:, 0] = -1
    assert S.pinned_runs(p) == ((0, 1), (2, 5), (9, 10))
    assert S.pinned_runs(p, return_logits=True) == ((0, 10),)
    assert S.pinned_runs(torch.zeros(3, 10, dtype=torch.int32), return_logits=True) == ((0, 10),)
    assert S.pinned_runs(torch.zeros(2, 0, dtype=torch.int32)) == ()


# ------------------------------------------------------------------------------ the pin rule
def _case(r, B, Tp_o, edits, V_=1024):
    """Originals of B rows and an edit (a, b, n) per row with one Tp_e: -> (phone, orig_phone, d, codes, span)."""
    d = torch.from_numpy(r.integers(1, 20, (B, Tp_o)))
    oph = torch.from_numpy(r.integers(0, 300, (B, Tp_o)))
    N_o = d.sum(1)
    codes = torch.from_numpy(r.integers(0, V_, (B, int(-(-N_o.max() // 8)) + 2)))
    rows = []
    for i, (a, b, n) in enumerate(edits):
        rows.append(torch.cat([oph[i, :a], torch.from_numpy(r.integers(300, 320, n)), oph[i, b:]]))
    assert len({len(x) for x in rows}) == 1
    return torch.stack(rows), oph, d, codes, torch.tensor([[a, b] for a, b, _ in edits])


def _check_rule(ph, oph, d, codes, span, new_frames):
    plan = EditPlan(ph, oph, d, codes, span, None, 1024)
    totals = [plan.F_a[r] + new_frames[r] + plan.F_s[r] for r in range(plan.B)]
    T = -(-max(totals) // 8)
    got = plan.code_pins(totals, T)
    want = RE.code_pins(d.tolist(), codes.tolist(), span.tolist(), plan.n, new_frames, T)
    assert torch.equal(got.long(), want), (span.tolist(), new_frames)
    assert plan.edit_frames(totals).tolist() == [[plan.F_a[r], plan.F_a[r] + new_frames[r]] for r in range(plan.B)]
    return plan, got, totals


@pytest.mark.parametrize("seed", range(12))
def test_pin_rule_equals_the_restatement_on_random_edits(seed):
    r = np.random.default_rng(seed)
    B, Tp_o = 4, int(r.integers(3, 30))
    dn = int(r.integers(-2, 4))
    edits = []
    for _ in range(B):
        while True:
            a = int(r.integers(0, Tp_o + 1))
            b = int(r.integers(a, Tp_o + 1))
            n = b - a + dn
            if n >= 0:
                break
            dn = max(dn, a - b)
        edits.append((a, b, n))
    edits = [(a, b, b - a + dn) for a, b, _ in edits if b - a + dn >= 0]
    while len(edits) < B:
        edits.append((0, Tp_o, Tp_o + dn))
    ph, oph, d, codes, span = _case(r, B, Tp_o, edits)
    L_n = [int(r.integers(n, 12 * n + 1)) if n else 0 for _, _, n in edits]
    _check_rule(ph, oph, d, codes, span, L_n)


def test_pin_rule_edges():
    r = np.random.default_rng(99)
    Tp = 12
    d = torch.from_numpy(r.integers(1, 20, (1, Tp)))
    oph = torch.from_numpy(r.integers(0, 300, (1, Tp)))
    N_o = int(d.sum())
    codes = torch.from_numpy(r.integers(0, 1024, (1, -(-N_o // 8))))

    def edit(a, b, n, L_n):
        ph = torch.cat([oph[0, :a], torch.arange(300, 300 + n), oph[0, b:]])[None]
        return _check_rule(ph, oph, d, codes, torch.tensor([[a, b]]), [L_n])

    plan, pins, _ = edit(0, Tp, 3, 20)                      # a = 0, b = Tp_o: every block is new
    assert (pins == -1).all()
    plan, pins, _ = edit(0, 0, 0, 0)                        # the identity edit: every step pinned to its own code
    assert torch.equal(pins.long(), codes)
    plan, pins, _ = edit(5, 5, 2, 11)                       # insertion
    assert plan.n == [2] and plan.L_o == [0]
    plan, pins, _ = edit(3, 6, 0, 0)                        # deletion
    L_o = plan.L_o[0]
    edit(3, 6, 1, L_o)                                      # span_frames = L_o: the suffix keeps its blocks
    for a in range(Tp):                                     # F_a % 8 zero and non-zero
        edit(a, a + 1, 1, 5)
    # a shift by a multiple of 8 keeps orig_codes[k - s / 8] exactly
    F_a = int(d[0, :4].sum())
    for L_n in (int(d[0, 4]) + 8, int(d[0, 4]) - 8 if int(d[0, 4]) > 8 else int(d[0, 4]) + 16):
        plan, pins, totals = edit(4, 5, 1, L_n)
        s = L_n - int(d[0, 4])
        assert s % 8 == 0
        for k in range(pins.shape[1]):
            if 8 * k >= F_a + L_n and 8 * k < totals[0]:
                assert int(pins[0, k]) == int(codes[0, k - s // 8])
    edit(4, 5, 1, 1)                                        # s < 0
    # ragged N_e across rows and a last partial block
    ph = torch.stack([torch.cat([oph[0, :2], torch.tensor([301, 302]), oph[0, 3:]]),
                      torch.cat([oph[0, :7], torch.tensor([303, 304]), oph[0, 8:]])])
    rest = N_o - int(d[0, 7])
    L_n1 = 30 + (5 - (rest + 30)) % 8                       # row 1 ends 5 frames into its last block
    _, pins, totals = _check_rule(ph, oph.repeat(2, 1), d.repeat(2, 1), codes.repeat(2, 1),
                                  torch.tensor([[2, 3], [7, 8]]), [3, L_n1])
    assert totals[0] != totals[1] and totals[1] % 8 == 5
    short = min(range(2), key=lambda i: totals[i])
    assert (pins[short, -(-totals[short] // 8):] == 0).all()


# ------------------------------------------------------------------------------ edit validation
def _tts():
    tts = Megatts.__new__(Megatts)
    torch.nn.Module.__init__(tts)
    tts.plm = _plm()
    return tts


def _orig():
    oph = torch.tensor([[10, 11, 12, 13, 14], [20, 21, 22, 23, 24]])
    d = torch.tensor([[3, 4, 5, 6, 7], [2, 2, 2, 2, 2]])
    codes = torch.zeros(2, 4, dtype=torch.int64)
    span = torch.tensor([[1, 3], [2, 4]])             # each row replaces 2 phones by 2 new ones
    ph = torch.tensor([[10, 97, 98, 13, 14], [20, 21, 98, 99, 24]])
    return ph, oph, d, codes, span


def test_edit_plan_of_a_valid_edit():
    ph, oph, d, codes, span = _orig()
    ph = torch.cat([ph, torch.tensor([[0], [0]])], 1)
    ph[0] = torch.tensor([10, 97, 98, 96, 13, 14])     # 3 new phones in row 0
    ph[1] = torch.tensor([20, 21, 98, 99, 22, 23])
    span = torch.tensor([[1, 3], [2, 3]])               # row 1: 2 new phones replace phone 2
    with pytest.raises(L.MttsError):                    # row 1's suffix is [23, 24], not [22, 23]
        EditPlan(ph, oph, d, codes, span, None, V)
    ph[1] = torch.tensor([20, 21, 98, 99, 23, 24])
    plan = EditPlan(ph, oph, d, codes, span, [6, 4], V)
    assert plan.n == [3, 2] and plan.F_a == [3, 4] and plan.L_o == [9, 2] and plan.F_s == [13, 4]
    assert plan.pinned_durations.tolist() == [[3, -1, -1, -1, 6, 7], [2, 2, -1, -1, 2, 2]]
    assert plan.total_frames.tolist() == [22, 12]


@pytest.mark.parametrize("change, match", [
    (dict(span=[[3, 1], [2, 4]]), r"span\[0\] = \[3, 1\)"),
    (dict(span=[[1, 3], [2, 6]]), r"span\[1\] = \[2, 6\)"),
    (dict(short=2), r"span\[0\] = \[1, 3\).*1 fewer"),
    (dict(prefix=(1, 0)), r"phone_tokens\[1, 0\] = 77 differs from orig_phone\[1, 0\]"),
    (dict(suffix=(0, 4)), r"phone_tokens\[0, 4\] = 77 differs from orig_phone\[0, 4\]"),
    (dict(dur=(0, 0, 0)), r"orig_durations\[0, 0\] = 0"),
    (dict(dur=(1, 4, 128)), r"orig_durations\[1, 4\] = 128"),
    (dict(dur=(0, 1, -1)), r"orig_durations\[0, 1\] = -1"),
    (dict(codes=3), r"orig_codes\[0\]: 3 codes"),
    (dict(code=(1, 1, V)), rf"orig_codes\[1, 1\] = {V}"),
    (dict(code=(0, 2, -1)), r"orig_codes\[0, 2\] = -1"),
    (dict(span_frames=[1, 4]), r"span_frames\[0\] = 1"),
    (dict(span_frames=[4, 257]), r"span_frames\[1\] = 257"),
    (dict(span_frames=[4]), r"span_frames: shape"),
    (dict(span=[[1, 3]]), r"expected orig_phone"),
])
def test_edit_rejects(change, match):
    ph, oph, d, codes, span = _orig()
    sf = None
    if "span" in change:
        span = torch.tensor(change["span"])
    if "short" in change:
        ph = ph[:, :change["short"]]
    if "prefix" in change:
        ph[change["prefix"]] = 77
    if "suffix" in change:
        ph[change["suffix"]] = 77
    if "dur" in change:
        r_, j, v = change["dur"]
        d[r_, j] = v
    if "codes" in change:
        codes = codes[:, :change["codes"]]
    if "code" in change:
        r_, j, v = change["code"]
        codes[r_, j] = v
    if "span_frames" in change:
        sf = change["span_frames"]
    with pytest.raises(L.MttsError, match=match):
        _tts().edit(ph, None, oph, d, codes, span, span_frames=sf)


def test_edit_accepts_a_replaced_duration_of_zero_and_128():
    ph, oph, d, codes, span = _orig()
    d[0, 1], d[0, 2] = 0, 128                          # replaced phones: any count a recording's aligner gives
    codes = torch.zeros(2, 20, dtype=torch.int64)
    EditPlan(ph, oph, d, codes, span, None, V)


@pytest.mark.parametrize("name", REJECTED)
def test_edit_rejects_synthesize_arguments_by_name(name):
    ph, oph, d, codes, span = _orig()
    with pytest.raises(L.MttsError, match=f"edit does not take {name}"):
        _tts().edit(ph, None, oph, d, codes, span, **{name: 1})
    with pytest.raises(TypeError):
        _tts().edit(ph, None, oph, d, codes, span, no_such_argument=1)


def test_edit_rejects_bad_controls_before_any_device_work():
    ph, oph, d, codes, span = _orig()
    with pytest.raises(L.MttsError, match="duration_scale"):
        _tts().edit(ph, None, oph, d, codes, span, duration_scale=0.0)


# ------------------------------------------------------------------------------ dispatch
class PinRecorder(Recorder):
    """The recorder, with the pinned entry's codes_out at its own position."""

    def _call(self, name, *args):
        if name != "mtts_plm_infer_pinned_f32":
            return super()._call(name, *args)
        types = L.SIGNATURES[name][1]
        assert len(args) == len(types)
        norm = [_norm(a, t) for a, t in zip(args, types)]
        norm[-2] = WS_OK if args[-2] >= 4096 else args[-2]
        self.calls.append((name, tuple(norm)))
        return 0


from test_plm_dispatch_host import _norm  # noqa: E402


@pytest.fixture
def plib(lib, monkeypatch):  # noqa: F811
    rec = PinRecorder()
    monkeypatch.setattr(L, "lib", lambda: rec)
    return rec


@pytest.mark.parametrize("rl", [False, True])
@pytest.mark.parametrize("sampled", [False, True])
def test_infer_without_pins_calls_what_it_called(plib, sampled, rl):
    _plm().infer(_latent(), return_logits=rl, pinned=None, **_smp(sampled))
    names = [n for n, _ in plib.calls]
    assert names == ["mtts_plm_infer_workspace_bytes",
                     "mtts_plm_infer_sample_f32" if sampled else "mtts_plm_infer_f32"]


@pytest.mark.parametrize("sampled", [False, True])
def test_pins_call_the_pinned_entry_once_per_run(plib, sampled):
    pins = torch.tensor([[3, -1, 4, 5, -1], [3, 2, 4, -1, -1]])
    codes = _plm().infer(_latent(), pinned=pins, **_smp(sampled))
    s = SMP_STRUCT if sampled else None
    base = (M_PLM, P, 48, 8, 2, 5, None, 0, 0, None, 0, 0)
    assert plib.calls == [
        ("mtts_plm_infer_ctx_workspace_bytes", (M_PLM, 2, 0, 5)),
        ("mtts_plm_infer_pinned_f32", base + (1, 2, P, P, None, s, P, 5, P, WS_OK, "stream")),
        ("mtts_plm_infer_pinned_f32", base + (3, 5, P, P, None, s, P, 5, P, WS_OK, "stream"))]
    # the recorder decodes nothing: the returned codes are the state built from BOS and the pins
    assert codes.shape == (2, 5) and codes[:, 0].tolist() == [3, 3] and codes[:, 2].tolist() == [4, 4]
    assert codes[0, 1] == V and codes[1, 1] == 2


def test_pins_with_logits_and_a_context(plib):
    ctx = PLMContext(torch.randn(1, 3, 8), torch.randint(0, V, (1, 3)))
    codes, logits = _plm().infer(_latent(), return_logits=True, context=ctx, pinned=torch.zeros(2, 5, dtype=torch.int32))
    assert plib.calls == [
        ("mtts_plm_infer_ctx_workspace_bytes", (M_PLM, 2, 3, 5)),
        ("mtts_plm_infer_pinned_f32", (M_PLM, P, 48, 8, 2, 5, P, 0, 8, P, 0, 3, 0, 5, P, P, P, None, P, 5, P, WS_OK,
                                       "stream"))]
    assert codes.tolist() == [[0] * 5] * 2 and logits.shape == (2, 5, V)


def test_all_pinned_enqueues_nothing(plib):
    codes = _plm().infer(_latent(), pinned=torch.full((2, 5), 7))
    assert plib.calls == [] and codes.tolist() == [[7] * 5] * 2


def test_other_decodes_reject_pins(plib):
    plm, pins = _plm(), torch.full((2, 5), -1)
    for call in (lambda: plm.infer_causal(_latent(), pinned=pins),
                 lambda: plm.infer_mix([_latent(), _latent()], [1.0, 1.0], pinned=pins),
                 lambda: plm.begin_decode(_latent(), pinned=pins)):
        with pytest.raises(L.MttsError, match="code pins"):
            call()
    with pytest.raises(L.MttsError, match="pinned codes"):
        plm.infer(_latent(), pinned=torch.full((2, 5), V))
    assert plib.calls == []


# ------------------------------------------------------------------------------ C side
def test_c_side_rejects_bad_pinned_arguments():
    """mtts_plm_infer_pinned_f32 validates before it enqueues anything (so no device is needed to see the errors)."""
    lib_ = L.lib()
    dummy = C.c_void_p(256)                    # never dereferenced: every call below fails its checks first
    layer = L.EncoderLayer()
    plm = L.PLM()
    plm.enc.layers = C.pointer(layer)
    plm.enc.d_model, plm.enc.n_heads, plm.vq_dim, plm.tc_dim, plm.vq_bins = 16, 2, 8, 8, 16
    plm.pc_embedding = plm.w_predict = plm.pe = 256

    def call(j0=0, j1=1, state=dummy, pin=dummy, pin_sb=4, m=C.byref(plm), ws=dummy, P_=0, ctx=None):
        return lib_.mtts_plm_infer_pinned_f32(m, dummy, 0, 8, 1, 4, ctx, 0, 8, ctx, 0, P_, j0, j1, state, dummy, None,
                                              None, pin, pin_sb, ws, 1 << 30, None)
    assert call(pin_sb=-1) == -1 and "pin_sb" in lib_.mtts_last_error().decode()
    assert call(j1=5) == -1                                # j1 > T
    assert call(j0=2, j1=1) == -1
    assert call(state=None) == -1 and call(m=None) == -1 and call(ws=None) == -1
    assert call(P_=2) == -1 and "context" in lib_.mtts_last_error().decode()
    bad = L.Sampling()
    bad.temperature = -1.0
    assert lib_.mtts_plm_infer_pinned_f32(C.byref(plm), dummy, 0, 8, 1, 4, None, 0, 8, None, 0, 0, 0, 1, dummy, dummy,
                                          None, C.byref(bad), dummy, 4, dummy, 1 << 30, None) == -1


def test_ctypes_signature_matches_the_header():
    src = open(os.path.join(ROOT, "include", "megatts2_b200.h")).read()
    name = "mtts_plm_infer_pinned_f32"
    m = re.search(r"\b" + name + r"\(([^)]*)\)", src)
    assert m
    assert len(L.SIGNATURES[name][1]) == len([a for a in m.group(1).split(",") if a.strip()])
    assert L.SIGNATURES[name][0] is C.c_int
    assert L.SIGNATURES[name][1][:18] == L.SIGNATURES["mtts_plm_infer_ctx_range_f32"][1][:18]
