"""CPU: which library entry points MegaPLM and MegaADM call, and with what.  The library is replaced by a recorder, so each
case pins the sequence of entries, their integer arguments, which pointers are NULL, the sampling struct, the output
shapes and the CUDA-graph caches the calls fill, without a device and without the built library."""
import ctypes as C
import functools

import pytest
import torch

from megatts2_b200 import _lib as L
from megatts2_b200 import graphs, ops, pack
from megatts2_b200.models.megatts2 import MegaADM, MegaPLM
from megatts2_b200.sampling import Sampling

WS = 4096                     # what every *_workspace_bytes query returns
STREAM = 0x5EA                # the stream handle the stubbed ops._stream() passes
P, M_PLM, M_ADM = "ptr", "plm", "adm"
WS_OK = "ws >= queried"
SMP = Sampling(temperature=0.7, top_k=5, top_p=0.9, seed=11)
SMP_STRUCT = ("sampling", C.c_float(0.7).value, 5, C.c_float(0.9).value, 0, 11, (7, 9))


def _code(b, t):
    """The code the recorder writes for utterance b at step t."""
    return 100 * b + t


def _codes(t0, t1):
    return torch.tensor([[_code(b, t) for t in range(t0, t1)] for b in range(2)], dtype=torch.int64)


class Recorder:
    """Stands in for the library: records (entry, normalised arguments) and returns WS for a workspace query, else 0.  A
    PLM decode entry also writes _code(b, t) into all of its (2, 5) codes_out, as if it had decoded every step."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return functools.partial(self._call, name)

    def _call(self, name, *args):
        types = L.SIGNATURES[name][1]
        assert len(args) == len(types), name
        query = name.endswith("_workspace_bytes")
        if name.startswith("mtts_plm_") and not query:
            codes = (C.c_int64 * 10).from_address(args[-6 if C.POINTER(L.Sampling) in types else -5])
            codes[:] = [_code(b, t) for b in range(2) for t in range(5)]
        norm = [_norm(a, t) for a, t in zip(args, types)]
        if not query:
            assert types[-2] is C.c_int64
            norm[-2] = WS_OK if args[-2] >= WS else args[-2]
        self.calls.append((name, tuple(norm)))
        return WS if query else 0


def _norm(a, t):
    if t in (C.c_int32, C.c_int64):
        assert isinstance(a, int)
        return a
    if t is C.c_void_p:
        v = a.value if isinstance(a, C.c_void_p) else a
        return None if not v else "stream" if v == STREAM else P
    if a is None:
        return None
    obj = a._obj                                   # a ctypes byref() argument
    if isinstance(obj, L.Sampling):
        return ("sampling", obj.temperature, obj.top_k, obj.top_p, obj.reserved,
                C.c_int64.from_address(obj.seed).value, tuple((C.c_int64 * 2).from_address(obj.keys)))
    return {L.PLM: M_PLM, L.ADM: M_ADM}[type(obj)]


def _stub_plan(self, device, T, struct):
    if self._plan is None:
        self._plan = pack.Plan()
        self._plan.struct = struct()
    return self._plan


@pytest.fixture
def lib(monkeypatch):
    rec = Recorder()
    monkeypatch.setattr(L, "lib", lambda: rec)

    def dev(t, dtype=torch.float32, name="tensor"):
        if not isinstance(t, torch.Tensor) or t.dtype != dtype:
            raise L.MttsError(f"{name}: expected a {dtype} tensor")
        return t
    monkeypatch.setattr(ops, "_dev", dev)
    monkeypatch.setattr(ops, "workspace", lambda nbytes, device: torch.empty(int(nbytes) + 256, dtype=torch.uint8,
                                                                             device=device))
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(STREAM))
    monkeypatch.setattr(MegaPLM, "_plan_get", lambda self, device, T: _stub_plan(self, device, T, L.PLM))
    monkeypatch.setattr(MegaADM, "_plan_get", lambda self, device, T: _stub_plan(self, device, T, L.ADM))
    monkeypatch.setattr(graphs, "_enabled", False)
    return rec


def _plm():
    return MegaPLM(n_layers=1, n_heads=2, vq_dim=8, tc_latent_dim=8, vq_bins=16).eval()


def _adm():
    return MegaADM(n_layers=1, n_heads=2, emb_dim=8, tc_latent_dim=8, tc_emb_dim=8).eval()


def _latent():
    """(2, 5, 8) with unit channel stride and batch stride 48: passed through as it is."""
    return torch.randn(2, 6, 8)[:, :5]


def _latent_t():
    """(2, 5, 8) with channel stride 5: made contiguous (strides 40, 8) before the call."""
    return torch.randn(2, 8, 5).transpose(1, 2)


def _smp(sampled):
    return dict(sampling=SMP, keys=[7, 9]) if sampled else {}


def _split(out, rl):
    return out if rl else (out, None)


@pytest.mark.parametrize("rl", [False, True])
@pytest.mark.parametrize("sampled", [False, True])
def test_infer(lib, sampled, rl):
    out = _plm().infer(_latent(), return_logits=rl, **_smp(sampled))
    lg = P if rl else None
    if sampled:
        call = ("mtts_plm_infer_sample_f32", (M_PLM, P, 48, 8, 2, 5, P, lg, SMP_STRUCT, P, WS_OK, "stream"))
    else:
        call = ("mtts_plm_infer_f32", (M_PLM, P, 48, 8, 2, 5, P, lg, P, WS_OK, "stream"))
    assert lib.calls == [("mtts_plm_infer_workspace_bytes", (M_PLM, 2, 5)), call]
    codes, logits = _split(out, rl)
    assert codes.dtype == torch.int64 and torch.equal(codes, _codes(0, 5))
    if rl:
        assert logits.shape == (2, 5, 16) and logits.dtype == torch.float32


@pytest.mark.parametrize("rl", [False, True])
@pytest.mark.parametrize("sampled", [False, True])
def test_infer_mix(lib, sampled, rl):
    out = _plm().infer_mix([_latent(), _latent()], [1.0, 3.0], return_logits=rl, **_smp(sampled))
    assert lib.calls == [
        ("mtts_plm_infer_mix_workspace_bytes", (M_PLM, 2, 2, 5)),
        ("mtts_plm_infer_mix_f32", (M_PLM, 2, P, 40, 8, 2, 5, P, P, P if rl else None, SMP_STRUCT if sampled else None,
                                    P, WS_OK, "stream"))]
    codes, logits = _split(out, rl)
    assert codes.dtype == torch.int64 and torch.equal(codes, _codes(0, 5))
    if rl:
        assert logits.shape == (2, 2, 5, 16) and logits.dtype == torch.float32


@pytest.mark.parametrize("rl", [False, True])
@pytest.mark.parametrize("sampled", [False, True])
@pytest.mark.parametrize("mixed", [False, True])
def test_decode_until(lib, mixed, sampled, rl):
    plm = _plm()
    if mixed:
        dec = plm.begin_decode([_latent(), _latent()], weights=[1.0, 3.0], **_smp(sampled))
    else:
        dec = plm.begin_decode(_latent(), **_smp(sampled))
    assert lib.calls == []
    outs = [plm.decode_until(dec, t1, return_logits=rl) for t1 in (2, 2, 5)]
    lg = P if rl else None

    def steps(t0, t1):
        if mixed:
            return [("mtts_plm_infer_mix_workspace_bytes", (M_PLM, 2, 2, 5)),
                    ("mtts_plm_infer_mix_range_f32", (M_PLM, 2, P, 40, 8, 2, 5, P, t0, t1, P, P, lg,
                                                      SMP_STRUCT if sampled else None, P, WS_OK, "stream"))]
        if sampled:
            call = ("mtts_plm_infer_range_sample_f32", (M_PLM, P, 48, 8, 2, 5, t0, t1, P, P, lg, SMP_STRUCT, P, WS_OK,
                                                        "stream"))
        else:
            call = ("mtts_plm_infer_range_f32", (M_PLM, P, 48, 8, 2, 5, t0, t1, P, P, lg, P, WS_OK, "stream"))
        return [("mtts_plm_infer_workspace_bytes", (M_PLM, 2, 5)), call]
    assert lib.calls == steps(0, 2) + steps(2, 5)         # the empty range [2, 2) calls nothing
    for out, (t0, t1) in zip(outs, [(0, 2), (2, 2), (2, 5)]):
        codes, logits = _split(out, rl)
        assert codes.dtype == torch.int64 and torch.equal(codes, _codes(t0, t1))
        if rl:
            assert logits.shape == ((2, 2, t1 - t0, 16) if mixed else (2, t1 - t0, 16))
            assert logits.dtype == torch.float32
    assert dec.t == 5 and torch.equal(dec.codes, _codes(0, 5)) and torch.equal(dec.state[:, 0], torch.tensor([16, 16]))


@pytest.mark.parametrize("rl", [False, True])
@pytest.mark.parametrize("sampled", [False, True])
def test_infer_causal(lib, sampled, rl):
    out = _plm().infer_causal(_latent_t(), return_logits=rl, **_smp(sampled))
    lg = P if rl else None
    if sampled:
        call = ("mtts_plm_decode_causal_sample_f32", (M_PLM, P, 40, 8, 2, 5, P, lg, SMP_STRUCT, P, WS_OK, "stream"))
    else:
        call = ("mtts_plm_decode_causal_f32", (M_PLM, P, 40, 8, 2, 5, P, lg, P, WS_OK, "stream"))
    assert lib.calls == [("mtts_plm_decode_causal_workspace_bytes", (M_PLM, 2, 5)), call]
    codes, logits = _split(out, rl)
    assert codes.dtype == torch.int64 and torch.equal(codes, _codes(0, 5))
    if rl:
        assert logits.shape == (2, 5, 16) and logits.dtype == torch.float32


@pytest.mark.parametrize("raw", [False, True])
@pytest.mark.parametrize("causal", [False, True])
def test_adm(lib, causal, raw):
    adm = _adm()
    if causal:
        out = adm.infer_causal(_latent_t(), return_raw=raw)
        calls = [("mtts_adm_decode_causal_workspace_bytes", (M_ADM, 2, 5)),
                 ("mtts_adm_decode_causal_f32", (M_ADM, P, 40, 8, 2, 5, P, P if raw else None, P, WS_OK, "stream"))]
    else:
        out = adm.infer(_latent(), return_raw=raw)
        calls = [("mtts_adm_infer_workspace_bytes", (M_ADM, 2, 5)),
                 ("mtts_adm_infer_f32", (M_ADM, P, 48, 8, 2, 5, P, P if raw else None, P, WS_OK, "stream"))]
    assert lib.calls == calls
    dur, r = out if raw else (out, None)
    assert dur.shape == (2, 5, 1) and dur.dtype == torch.int32
    if raw:
        assert r.shape == (2, 5) and r.dtype == torch.float32


def _graph_caches(d):
    """The GraphedCall objects held by a module's __dict__ (or its pickled state), directly or in a dict."""
    found = []
    for v in d.values():
        found += [x for x in (v.values() if isinstance(v, dict) else [v]) if isinstance(x, graphs.GraphedCall)]
    return found


def test_graph_caches(lib, monkeypatch):
    """Whole decodes share the module's main cache; ranges go to a cache of their own; neither is pickled.  Each key is
    called once only: a second call would capture."""
    monkeypatch.setattr(graphs, "_enabled", True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    plm = _plm()
    main = plm._graphs()
    plm.infer(_latent())
    assert len(main.cache) == 1
    plm.infer(_latent(), **_smp(True))
    assert len(main.cache) == 2
    plm.infer_mix([_latent(), _latent()], [1.0, 3.0])
    assert len(main.cache) == 3
    dec = plm.begin_decode(_latent())
    plm.decode_until(dec, 2)
    plm.decode_until(dec, 5)
    assert len(main.cache) == 3
    others = [g for g in _graph_caches(plm.__dict__) if g is not main]
    assert sum(len(g.cache) for g in others) == 2
    assert _graph_caches(plm.__getstate__()) == []
