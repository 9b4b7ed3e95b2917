"""CPU: the prosody LM's in-context decode on the host - identities of its restatement (tests/ref_plm_context.py), the
PLMContext checks, the entry points MegaPLM calls with a context (the library replaced by the recorder of
test_plm_dispatch_host), the rejected combinations, the C side's argument checks and the ctypes mirror of the new entries."""
import ctypes as C
import re

import pytest
import torch

import ref_plm_context as PC
from conftest import ROOT
from megatts2_b200 import _lib as L
from megatts2_b200.models.megatts2 import Megatts, PLMContext, _context_inputs
from oracle import ref_megatts2 as R
from oracle import weights
from test_plm_dispatch_host import M_PLM, P, SMP_STRUCT, WS_OK, _latent, _plm, _smp, lib  # noqa: F401  (lib: the fixture)

CFG = weights.PLM_CFG


def gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def sd():
    return weights.plm_state_dict()


def ctx_of(Bc, P_, seed):
    return (torch.randn(Bc, P_, 512, generator=gen(seed)).abs(),
            torch.randint(0, CFG["vq_bins"], (Bc, P_), generator=gen(seed + 1)))


# ------------------------------------------------------------------------------ restatement identities
@pytest.mark.parametrize("causal", [False, True])
def test_empty_context_is_the_plain_decode(sd, causal):
    tc = torch.randn(2, 4, 512, generator=gen(3)).abs()
    ctx_tc, ctx_codes = ctx_of(1, 0, 5)
    codes, logits = PC.plm_infer_ctx(sd, ctx_tc, ctx_codes, tc, CFG, causal=causal, return_logits=True)
    ref = (R.plm_infer_causal if causal else R.plm_infer)(R.SD(sd), tc, CFG, return_logits=True)
    assert torch.equal(codes, ref[0]) and torch.equal(logits, ref[1])


@pytest.mark.parametrize("Bc", [1, 2])
def test_causal_restatement_is_the_teacher_forced_forward(sd, Bc):
    """Each step's logits are the last row of R.plm_forward over its prefix; one R.plm_forward over [context; target] at the
    decoded codes gives them all, within fp32 rounding (the two evaluate the same causal rows in differently sized GEMMs)."""
    tc = torch.randn(2, 5, 512, generator=gen(11)).abs()
    ctx_tc, ctx_codes = ctx_of(Bc, 6, 13)
    codes, logits = PC.plm_infer_ctx(sd, ctx_tc, ctx_codes, tc, CFG, causal=True, return_logits=True)
    whole = PC.causal_logits_on(sd, ctx_tc, ctx_codes, tc, codes, CFG)
    assert (whole - logits).abs().max().item() <= 1e-4


def test_context_is_the_teacher_forced_concatenation(sd):
    """Step j of the non-causal restatement is R.plm_step_logits over cat(ctx, target) with the context codes forced; a
    Bc = 1 context equals the same context repeated over B; the fp64 restatement is close to the fp32 one."""
    tc = torch.randn(2, 3, 512, generator=gen(21)).abs()
    ctx_tc, ctx_codes = ctx_of(1, 4, 23)
    codes, logits = PC.plm_infer_ctx(sd, ctx_tc, ctx_codes, tc, CFG, return_logits=True)
    rep = PC.plm_infer_ctx(sd, ctx_tc.expand(2, -1, -1), ctx_codes.expand(2, -1), tc, CFG, return_logits=True)
    assert torch.equal(codes, rep[0]) and torch.equal(logits, rep[1])
    lat = torch.cat([ctx_tc.expand(2, -1, -1), tc], 1)
    hist = torch.cat([torch.full((2, 1), CFG["vq_bins"]), ctx_codes.expand(2, -1), codes], 1)
    for j in range(3):
        want = R.plm_step_logits(R.SD(sd), lat, hist[:, :4 + j + 1], CFG)
        assert torch.equal(logits[:, j], want), j
    sd64 = PC.sd_as(sd, torch.float64)
    c64, l64 = PC.plm_infer_ctx(sd64, ctx_tc.double(), ctx_codes, tc.double(), CFG, return_logits=True)
    assert l64.dtype == torch.float64 and (l64 - logits.double()).abs().max().item() <= 1e-3


def test_sampled_steps_are_keyed_by_the_target_step(sd):
    """A sampled draw at target step j uses the noise of step j, not of position P + j: the restatement's picks equal the
    sampler's oracle at step j on its own logits."""
    from oracle import ref_sampling as RS
    tc = torch.randn(2, 3, 512, generator=gen(31)).abs()
    ctx_tc, ctx_codes = ctx_of(2, 5, 33)
    smp = (0.9, 20, 1.0, 77)
    codes, logits = PC.plm_infer_ctx(sd, ctx_tc, ctx_codes, tc, CFG, sampling=smp, keys=[4, 8], return_logits=True)
    for j in range(3):
        picks, _ = RS.sample_rows(logits[:, j].numpy(), j, *smp, [4, 8])
        assert picks.tolist() == codes[:, j].tolist(), j


# ------------------------------------------------------------------------------ PLMContext
def test_plm_context_rejects_malformed_input():
    good_tc, good_codes = torch.zeros(1, 3, 8), torch.zeros(1, 3, dtype=torch.int64)
    for tc8, codes in ((good_tc.double(), good_codes), (good_tc, good_codes.int()), ("x", good_codes),
                       (torch.zeros(3, 8), good_codes), (good_tc, torch.zeros(1, 4, dtype=torch.int64)),
                       (good_tc, torch.zeros(3, dtype=torch.int64)), (torch.zeros(0, 3, 8), torch.zeros(0, 3).long()),
                       (good_tc, torch.tensor([[0, -1, 2]]))):
        with pytest.raises(L.MttsError, match="PLMContext"):
            PLMContext(tc8, codes)
    with pytest.raises(L.MttsError, match="CUDA"):                  # well-formed, but no CPU fallback
        PLMContext(good_tc, good_codes)


def test_contexts_join_in_order_and_are_checked_at_use(lib):  # noqa: F811  (ops._dev stubbed: CPU tensors stand in)
    a = PLMContext(torch.randn(1, 2, 8), torch.tensor([[1, 2]]))
    b = PLMContext(torch.randn(3, 4, 8), torch.arange(12).reshape(3, 4))
    j = PLMContext.cat([a, b])
    assert j.P == 6 and j.max_code == 11
    assert torch.equal(j.tc8, torch.cat([a.tc8.expand(3, -1, -1), b.tc8], 1))
    assert torch.equal(j.codes, torch.cat([a.codes.expand(3, -1), b.codes], 1))
    cpu = torch.device("cpu")
    tc8, codes = _context_inputs([a, b], 3, 8, 16, cpu)
    assert torch.equal(tc8, j.tc8) and torch.equal(codes, j.codes)
    assert _context_inputs(a, 5, 8, 16, cpu)[0].shape == (1, 2, 8)     # Bc = 1 serves any B
    for ctx, B, dim, V in ((b, 2, 8, 16), (a, 1, 9, 16), (b, 3, 8, 11), ([a, PLMContext(torch.zeros(2, 1, 8),
                                                                                        torch.zeros(2, 1).long()), b],
                                                                           3, 8, 16), ([], 1, 8, 16)):
        with pytest.raises(L.MttsError):
            _context_inputs(ctx, B, dim, V, cpu)


# ------------------------------------------------------------------------------ dispatch
def _ctx(Bc):
    return PLMContext(torch.randn(Bc, 3, 8), torch.randint(0, 16, (Bc, 3)))


@pytest.mark.parametrize("Bc", [1, 2])
@pytest.mark.parametrize("sampled", [False, True])
def test_infer_with_a_context_calls(lib, Bc, sampled):  # noqa: F811
    """One workspace query over P + T positions, one context decode; a Bc = 1 context has batch strides 0."""
    codes, logits = _plm().infer(_latent(), return_logits=True, context=_ctx(Bc), **_smp(sampled))
    sb = 0 if Bc == 1 else 24
    csb = 0 if Bc == 1 else 3
    assert lib.calls == [
        ("mtts_plm_infer_ctx_workspace_bytes", (M_PLM, 2, 3, 5)),
        ("mtts_plm_infer_ctx_f32", (M_PLM, P, 48, 8, 2, 5, P, sb, 8, P, csb, 3, P, P, SMP_STRUCT if sampled else None, P,
                                    WS_OK, "stream"))]
    assert codes.shape == (2, 5) and logits.shape == (2, 5, 16)


@pytest.mark.parametrize("sampled", [False, True])
def test_infer_causal_with_a_context_calls(lib, sampled):  # noqa: F811
    codes = _plm().infer_causal(_latent(), context=[_ctx(1), _ctx(2)], **_smp(sampled))
    assert lib.calls == [
        ("mtts_plm_decode_causal_ctx_workspace_bytes", (M_PLM, 2, 6, 5)),
        ("mtts_plm_decode_causal_ctx_f32", (M_PLM, P, 48, 8, 2, 5, P, 48, 8, P, 6, 6, P, None,
                                            SMP_STRUCT if sampled else None, P, WS_OK, "stream"))]
    assert codes.shape == (2, 5)


def test_ranges_with_a_context(lib):  # noqa: F811
    """The state is (B, P+T+1) with the context codes in columns 1..P from the start; decode_until stays in target steps
    and writes the target view."""
    plm, ctx = _plm(), _ctx(1)
    dec = plm.begin_decode(_latent(), context=ctx)
    assert dec.state.shape == (2, 3 + 5 + 1) and dec.P == 3
    assert torch.equal(dec.state[:, 0], torch.full((2,), 16)) and torch.equal(dec.state[:, 1:4], ctx.codes.expand(2, -1))
    c = plm.decode_until(dec, 2)
    assert c.shape == (2, 2) and torch.equal(dec.codes, c) and torch.equal(dec.target[:, :2], c)
    plm.decode_until(dec, 5)
    assert [n for n, _ in lib.calls] == ["mtts_plm_infer_ctx_workspace_bytes", "mtts_plm_infer_ctx_range_f32"] * 2
    assert lib.calls[1][1][12:14] == (0, 2) and lib.calls[3][1][12:14] == (2, 5)
    assert torch.equal(dec.state[:, 1:4], ctx.codes.expand(2, -1))        # the context columns are left alone
    with pytest.raises(L.MttsError):
        plm.begin_decode([_latent(), _latent()], weights=[1.0, 1.0], context=ctx)


def test_synthesize_rejects_a_context_with_prosody_prompts():
    tts = Megatts.__new__(Megatts)
    phone = torch.zeros(2, 3, dtype=torch.int64)
    with pytest.raises(L.MttsError, match="plm_context"):
        tts._check_prosody(phone, [torch.zeros(2, 4, 80)], [1.0, 1.0], False, None, plm_context=object())
    tts._check_prosody(phone, None, None, True, None, plm_context=object())        # the causal decode takes a context
    with pytest.raises(L.MttsError, match="PLM context"):
        tts.synthesize_many([(phone[0], torch.zeros(4, 80))], plm_context=object())


# ------------------------------------------------------------------------------ C side
def test_c_side_rejects_bad_contexts():
    """The context entries validate before they enqueue anything (so no device is needed to see the errors)."""
    lib_ = L.lib()
    dummy = C.c_void_p(256)                    # never dereferenced: every call below fails its checks first
    layer = L.EncoderLayer()
    plm = L.PLM()
    plm.enc.layers = C.pointer(layer)
    plm.enc.d_model, plm.enc.n_heads, plm.vq_dim, plm.tc_dim, plm.vq_bins = 16, 2, 8, 8, 16
    plm.pc_embedding = plm.w_predict = plm.pe = 256

    def infer(P_, ctx_tc=dummy, ctx_codes=dummy):
        return lib_.mtts_plm_infer_ctx_f32(C.byref(plm), dummy, 0, 8, 1, 1, ctx_tc, 0, 8, ctx_codes, 0, P_, dummy, None,
                                           None, dummy, 1 << 30, None)

    def causal(P_, ctx_tc=dummy, ctx_codes=dummy):
        return lib_.mtts_plm_decode_causal_ctx_f32(C.byref(plm), dummy, 0, 8, 1, 1, ctx_tc, 0, 8, ctx_codes, 0, P_, dummy,
                                                   None, None, dummy, 1 << 30, None)
    for call in (infer, causal):
        assert call(-1) == -1 and "context" in lib_.mtts_last_error().decode()
        assert call(2, ctx_tc=None) == -1 and "context" in lib_.mtts_last_error().decode()
        assert call(2, ctx_codes=None) == -1
    assert lib_.mtts_plm_infer_ctx_range_f32(C.byref(plm), dummy, 0, 8, 1, 4, dummy, 0, 8, dummy, 0, 2, 1, 5, dummy, dummy,
                                             None, None, dummy, 1 << 30, None) == -1       # j1 > T
    assert lib_.mtts_plm_infer_ctx_range_f32(C.byref(plm), dummy, 0, 8, 1, 4, dummy, 0, 8, dummy, 0, 2, 0, 1, None, dummy,
                                             None, None, dummy, 1 << 30, None) == -1       # no state
    m = C.byref(plm)
    assert lib_.mtts_plm_infer_ctx_workspace_bytes(m, 2, 0, 8) == lib_.mtts_plm_infer_workspace_bytes(m, 2, 8)
    assert lib_.mtts_plm_infer_ctx_workspace_bytes(m, 2, 5, 8) == lib_.mtts_plm_infer_workspace_bytes(m, 2, 13)
    assert lib_.mtts_plm_decode_causal_ctx_workspace_bytes(m, 2, 0, 8) == lib_.mtts_plm_decode_causal_workspace_bytes(
        m, 2, 8)
    assert lib_.mtts_plm_decode_causal_ctx_workspace_bytes(m, 2, 5, 8) > lib_.mtts_plm_decode_causal_workspace_bytes(
        m, 2, 13)


def test_ctypes_signatures_match_the_header():
    """Argument counts of the new entry points in _lib.SIGNATURES against their prototypes in the C header."""
    import os
    src = open(os.path.join(ROOT, "include", "megatts2_b200.h")).read()
    for name in ("mtts_plm_infer_ctx_workspace_bytes", "mtts_plm_infer_ctx_f32", "mtts_plm_infer_ctx_range_f32",
                 "mtts_plm_decode_causal_ctx_workspace_bytes", "mtts_plm_decode_causal_ctx_f32"):
        m = re.search(r"\b" + name + r"\(([^)]*)\)", src)
        assert m, name
        n_args = len([a for a in m.group(1).split(",") if a.strip()])
        assert len(L.SIGNATURES[name][1]) == n_args, name
        assert L.SIGNATURES[name][0] is (C.c_int64 if name.endswith("_bytes") else C.c_int), name
