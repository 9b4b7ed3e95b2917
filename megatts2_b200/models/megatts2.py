"""MegaG / MegaPLM / MegaADM / Megatts with the reference's surface (models/megatts2.py:30-117,
120-198, 201-292, 295-375) + a HiFi-GAN vocoder with speechbrain's ``HIFIGAN`` call surface
(``from_hparams`` / ``decode_batch``; reference call sites models/megatts2.py:321-323, 370-372).

Same class names, ctor kwargs, state_dict keys, ``forward`` / ``infer`` / ``from_hparams`` /
``from_pretrained`` signatures; all device work in libmegatts2_b200.  Differences, all
generalisations: ``infer`` accepts B >= 1 (B independent batch-1 runs of the reference, which is
hard-wired to B = 1 at :170-171, :262-263); ``Megatts.synthesize`` is the tensor-level body of
``Megatts.forward`` (:353-373) for a batch of utterances."""
import ctypes as C
import glob
import math

import torch
import torch.nn as nn
import yaml

from .. import _lib as L
from .. import autograd as A
from .. import ops, pack
from .. import edit as ED
from .. import passage as PS
from .. import sampling as S
from ..modules.convnet import ConvNet
from ..modules.embedding import SinePositionalEmbedding
from ..modules.mrte import MRTE, LengthRegulator, check_prompts
from ..modules.tokenizer import HIFIGAN_HOP_LENGTH, HIFIGAN_SR, extract_mel_spec
from ..modules.transformer import TransformerEncoder, TransformerEncoderLayer, encoder_plan, run_encoder
from ..modules.vqpe import VQProsodyEncoder
from ..utils.utils import instantiate_class


def _eval_only(m):
    if m.training:
        raise L.MttsError("this entry point is inference-only (call .eval()); training-mode forwards exist for MegaPLM / "
                          "MegaADM (SURVEY.md 8f-4), the generator trainer's path (conv stacks, VQ EMA) is not built")


def _dev_rows(t, name):
    """A CUDA fp32 (B, T, C) input with unit channel stride: ``t`` itself, or a contiguous copy."""
    t = ops._dev(t, name=name)
    return t if t.stride(2) == 1 else t.contiguous()


def _sampling_inputs(sampling, keys, rows, device):
    """(sampling, seed, keys) of a sampled decode, with the seed and the row keys as device tensors; None when greedy."""
    if sampling is None:
        return None
    return sampling, sampling.seed_tensor(device), S.row_keys(keys, rows, device)


def _mix_sources(tc_latents, weights, dim, what):
    """K source latents, each (B, T, dim), and their weights -> (the (K*B, T, dim) stack, (B, K) device weights, or
    (B, T, K) when ``weights`` is a schedule with one row per step).  ``what`` names the mix in the error messages."""
    if isinstance(tc_latents, torch.Tensor) or not len(tc_latents):
        raise L.MttsError(f"{what}: tc_latents must be a non-empty list of (B, T, tc_dim) tensors")
    tcs = [ops._dev(t, name=f"tc_latents[{k}]") for k, t in enumerate(tc_latents)]
    shape = tuple(tcs[0].shape)
    if len(shape) != 3 or shape[2] != dim or any(tuple(t.shape) != shape for t in tcs):
        raise L.MttsError(f"{what}: every source must be (B, T, {dim}) with the same B and T, got "
                          f"{[tuple(t.shape) for t in tcs]}")
    if any(t.device != tcs[0].device for t in tcs):
        raise L.MttsError(f"{what}: the sources must be on one device")
    if S.per_step(weights):
        w = S.mix_step_weights(weights, len(tcs), shape[0], shape[1], what)
    else:
        w = S.mix_weights(weights, len(tcs), shape[0], what)
    return torch.cat(tcs, 0), w.to(tcs[0].device)


class PLMContext:
    """A prompt context for the prosody LM's in-context decode (include/megatts2_b200.h states the contract): P rows of
    latents ``tc8`` (Bc, P, tc_dim) fp32 and their codes ``codes`` (Bc, P) int64 >= 0, on one CUDA device.  Bc is 1 (one
    context for every utterance of a call) or the call's batch size.  This is what the reference's MegaPLMDataset prepends
    to a target: a same-speaker cut's max-pooled MRTE latent and its VQ codes (``MegaG.plm_context`` makes one).  A list of
    contexts, wherever one is taken, is joined along P in the order given (``PLMContext.cat``).  The codes are read to the
    host once, here; the decode checks that they are below its ``vq_bins`` and that Bc fits its batch."""

    def __init__(self, tc8, codes):
        if not (isinstance(tc8, torch.Tensor) and tc8.dtype == torch.float32 and isinstance(codes, torch.Tensor)
                and codes.dtype == torch.int64):
            raise L.MttsError("PLMContext: tc8 must be a float32 tensor and codes an int64 tensor")
        if tc8.dim() != 3 or codes.dim() != 2 or codes.shape != tc8.shape[:2] or tc8.shape[0] < 1:
            raise L.MttsError(f"PLMContext: tc8 (Bc, P, tc_dim) and codes (Bc, P) with equal Bc >= 1 and P, got "
                              f"{tuple(tc8.shape)} and {tuple(codes.shape)}")
        if codes.device != tc8.device:
            raise L.MttsError("PLMContext: tc8 and codes must be on one device")
        lo, hi = torch.stack([codes.min(), codes.max()]).tolist() if codes.numel() else (0, -1)   # the one host read
        if lo < 0:
            raise L.MttsError(f"PLMContext: codes must be >= 0, got {lo}")
        ops._dev(tc8, name="PLMContext.tc8")
        self.tc8, self.codes, self.max_code = tc8.contiguous(), codes.contiguous(), hi

    @property
    def P(self):
        return self.tc8.shape[1]

    @staticmethod
    def from_rows(tc8, codes, max_code) -> "PLMContext":
        """A context from device rows whose codes are known to be in [0, max_code] (the prosody LM's own codes, or a
        checked context's), without the host read of ``__init__``."""
        out = PLMContext.__new__(PLMContext)
        out.tc8, out.codes, out.max_code = tc8.contiguous(), codes.contiguous(), max_code
        return out

    @staticmethod
    def cat(contexts) -> "PLMContext":
        """Contexts joined along P in the order given (their Bc all equal, or 1 and one other value)."""
        cs = list(contexts)
        if not cs or not all(isinstance(c, PLMContext) for c in cs):
            raise L.MttsError("PLMContext.cat: expected a non-empty list of PLMContext")
        if len(cs) == 1:
            return cs[0]
        Bc = max(c.tc8.shape[0] for c in cs)
        if any(c.tc8.shape[0] not in (1, Bc) for c in cs) or len({c.tc8.shape[2] for c in cs}) != 1:
            raise L.MttsError(f"PLMContext.cat: every Bc must be 1 or {Bc}, with one tc_dim")
        if len({c.tc8.device for c in cs}) != 1:
            raise L.MttsError("PLMContext.cat: the contexts must be on one device")
        out = PLMContext.__new__(PLMContext)
        out.tc8 = torch.cat([c.tc8.expand(Bc, -1, -1) for c in cs], 1).contiguous()
        out.codes = torch.cat([c.codes.expand(Bc, -1) for c in cs], 1).contiguous()
        out.max_code = max(c.max_code for c in cs)
        return out


def _context_inputs(context, B, tc_dim, vq_bins, device):
    """``context`` (a PLMContext, a list of them, or None) checked against a decode of B utterances -> (tc8 (Bc, P, tc_dim),
    codes (Bc, P)), or None."""
    if context is None:
        return None
    c = PLMContext.cat(context if isinstance(context, (list, tuple)) else [context])
    if c.tc8.shape[0] not in (1, B):
        raise L.MttsError(f"context: Bc = {c.tc8.shape[0]}, expected 1 or B = {B}")
    if c.tc8.shape[2] != tc_dim or c.tc8.device != device:
        raise L.MttsError(f"context: latents (Bc, P, {tc_dim}) on {device}, got {tuple(c.tc8.shape)} on {c.tc8.device}")
    if c.max_code >= vq_bins:
        raise L.MttsError(f"context: codes must be in [0, {vq_bins}), got {c.max_code}")
    return c.tc8, c.codes


def _ctx_args(ctx):
    """The context arguments of the mtts_plm_*_ctx_* entries; a batch stride of 0 broadcasts a Bc = 1 context."""
    tc8, codes = ctx
    one = tc8.shape[0] == 1
    return (tc8.data_ptr(), 0 if one else tc8.stride(0), tc8.stride(1), codes.data_ptr(), 0 if one else codes.stride(0),
            tc8.shape[1])


def _no_code_pins(pinned, what):
    if pinned is not None:
        raise L.MttsError(f"{what} does not take code pins: they are built for MegaPLM.infer's decode only")


def _ar_plan(model, enc, pos, struct, device, T, fill):
    """The weight plan of an AR model (MegaPLM / MegaADM), rebuilt when its weights or engine changed or when its
    positional table has fewer than T rows: the encoder ``enc``, then ``fill(plan, s)`` for the model's own fields of the
    ctypes ``struct``, then the table of ``pos`` with max(T, 4000) rows."""
    sig = pack.signature(list(model.parameters())) + (getattr(enc, "engine", None), pack.default_engine())
    if model._plan is None or model._plan.sig != sig or model._plan.pe_rows < T:
        pl = pack.Plan()
        pl.sig = sig
        enc_pl = encoder_plan(enc, list(enc.layers))
        pl.hold(enc_pl)
        s = struct()
        s.enc = enc_pl.enc
        fill(pl, s)
        pe = pos.table(device, max(T, 4000))
        pl.pe_rows = pe.shape[0]
        s.pe = pl.p(pe)
        s.pe_alpha = pos.alpha_host()
        pl.struct = s
        model._plan = pl
    return model._plan


class MegaG(nn.Module):
    def __init__(self, mrte: MRTE, vqpe: VQProsodyEncoder, kernel_size: int = 5, activation: str = 'ReLU',
                 hidden_size: int = 512, decoder_n_stack: int = 4, decoder_n_block: int = 2):
        super().__init__()
        self.mrte = mrte
        self.vqpe = vqpe
        self.decoder = ConvNet(
            in_channels=mrte.hidden_size + vqpe.vq.dimension, out_channels=mrte.mel_bins, hidden_size=hidden_size,
            n_stacks=decoder_n_stack, n_blocks=decoder_n_block, kernel_size=kernel_size, activation=activation)

    def forward(self, duration_tokens, phone, phone_lens, mel_mrte, mel_vqpe):
        """(models/megatts2.py:56-74; the reference raises TypeError here at this commit, SURVEY.md §0)."""
        _eval_only(self)
        zq, commit_loss, vq_loss, _ = self.vqpe(mel_vqpe)
        x = self.mrte(duration_tokens, phone, phone_lens, mel_mrte)
        T = min(x.shape[1], zq.shape[1])
        xin = torch.cat([x[:, :T], zq[:, :T]], dim=-1)
        return self.decoder.forward_cl(xin), commit_loss, vq_loss

    def s2_latent(self, phone, phone_lens, mel_mrte, mel_vqpe):
        """(models/megatts2.py:76-84)"""
        _, _, _, codes = self.vqpe(mel_vqpe)
        return self.mrte.tc_latent(phone, phone_lens, mel_mrte), codes

    def plm_context(self, phone, durations, mel_prompt, mel_timbre) -> PLMContext:
        """The prosody LM context of prompt utterances: the reference dataset's ``read_latent`` (modules/datamodule.py:
        163-178) applied to ``s2_latent``'s output, on the device.  phone (B, Tp) int64, durations (B, Tp) int, the
        utterances' mel ``mel_prompt`` (B, Tm, mel_bins) and the timbre mel ``mel_timbre`` (B, Tt, mel_bins).  The latent
        is ``mrte.tc_latent(phone, mel_timbre)`` length-regulated by ``durations`` and max-pooled by 8 (ceil); the codes are
        the VQ prosody encoder's codes of ``mel_prompt[:, :sum(d)]``; both have ceil(sum(d) / 8) rows.  Every utterance
        must have the same sum(d) (one host read), and mel_prompt at least that many frames."""
        _eval_only(self)
        d = torch.as_tensor(durations).to(phone.device, torch.int32)
        tc = self.mrte.tc_latent(phone, mel_timbre)
        tce, totals = ops.length_regulate(tc, d, return_host_totals=True)
        if len(set(totals)) > 1:
            raise L.MttsError(f"plm_context: every utterance needs the same sum(durations), got {totals}")
        n = totals[0] if totals else 0
        if mel_prompt.dim() != 3 or mel_prompt.shape[0] != phone.shape[0] or mel_prompt.shape[1] < n:
            raise L.MttsError(f"plm_context: mel_prompt ({phone.shape[0]}, >= {n}, mel_bins) needed, got "
                              f"{tuple(mel_prompt.shape)}")
        if n == 0:
            raise L.MttsError("plm_context: the durations sum to zero frames")
        _, _, _, codes = self.vqpe(mel_prompt[:, :n].contiguous())
        return PLMContext(ops.maxpool_time(tce, 8), codes[0])

    def decode_mel_cl(self, tc_latent_expand: torch.Tensor, p_codes: torch.Tensor) -> torch.Tensor:
        """Glue of Megatts.forward (models/megatts2.py:361-368): codes -> codebook rows repeated x8,
        truncated, concatenated with the expanded tc latent, then the ConvNet mel decoder.
        tc_latent_expand (B,L,512), p_codes (B,T8) int64 -> mel (B,L,80) channels-last."""
        B, Lm, H = tc_latent_expand.shape
        D = self.vqpe.vq.dimension
        x = torch.empty(B, Lm, H + D, dtype=torch.float32, device=tc_latent_expand.device)
        x[:, :, :H].copy_(tc_latent_expand)                       # layout plumbing (concat)
        embed = self.vqpe.vq.vq.layers[0]._codebook.embed
        ops.vq_gather(p_codes, embed, t_out=Lm, repeat=8, out=x[:, :, H:])
        return self.decoder.forward_cl(x)

    @classmethod
    def from_hparams(cls, config_path: str) -> "MegaG":
        with open(config_path, "r") as f:
            config = yaml.safe_load(f)
        g_cfg = config['model']['G']
        g_cfg['init_args']['mrte'] = instantiate_class(args=(), init=g_cfg['init_args']['mrte'])
        g_cfg['init_args']['vqpe'] = instantiate_class(args=(), init=g_cfg['init_args']['vqpe'])
        return instantiate_class(args=(), init=g_cfg)

    @classmethod
    def from_pretrained(cls, ckpt: str, config: str) -> "MegaG":
        G = cls.from_hparams(config)
        sd = {k[2:]: v for k, v in torch.load(ckpt, map_location="cpu")['state_dict'].items() if k.startswith('G.')}
        G.load_state_dict(sd, strict=True)
        return G


class MegaPLM(pack.PlanMixin, nn.Module):
    def __init__(self, n_layers: int = 12, n_heads: int = 16, vq_dim: int = 512, tc_latent_dim: int = 512,
                 vq_bins: int = 1024, dropout: float = 0.1):
        super().__init__()
        d_model = vq_dim + tc_latent_dim
        self.plm = TransformerEncoder(
            TransformerEncoderLayer(dim=d_model, ff_dim=d_model * 4, n_heads=n_heads, dropout=dropout, conv_ff=False),
            num_layers=n_layers)
        self.predict_layer = nn.Linear(d_model, vq_bins, bias=False)
        self.pos = SinePositionalEmbedding(d_model)
        self.pc_embedding = nn.Embedding(vq_bins + 2, vq_dim)
        self.vq_bins, self.vq_dim, self.tc_latent_dim = vq_bins, vq_dim, tc_latent_dim
        self._plan = None

    def _plan_get(self, device, T):
        def fill(pl, s):
            s.pc_embedding = pl.p(self.pc_embedding.weight)
            s.w_predict = pl.p(pack.pack_linear(self.predict_layer.weight))
            s.vq_bins, s.vq_dim, s.tc_dim = self.vq_bins, self.vq_dim, self.tc_latent_dim
        return _ar_plan(self, self.plm, self.pos, L.PLM, device, T, fill)

    def forward(self, tc_latent: torch.Tensor, p_codes: torch.Tensor, lens: torch.Tensor):
        """Teacher-forced logits with the causal + padding mask (models/megatts2.py:148-163).  In training mode the
        graph is built from megatts2_b200.autograd Functions (forward + backward kernels; SURVEY.md 8f-4)."""
        if self.training:
            pc_emb = A.EmbeddingFn.apply(p_codes[:, :-1], self.pc_embedding.weight)
            x = self.pos(torch.cat([tc_latent, pc_emb], dim=-1))
            h = self.plm(x, lens, causal=True)
            return A.linear(h, self.predict_layer.weight, None), p_codes[:, 1:]
        T = tc_latent.shape[1]
        dev = tc_latent.device
        x = torch.empty(tc_latent.shape[0], T, self.tc_latent_dim + self.vq_dim, dtype=torch.float32, device=dev)
        x[..., :self.tc_latent_dim].copy_(tc_latent)
        x[..., self.tc_latent_dim:].copy_(ops.embed_pe(p_codes[:, :-1].contiguous(), self.pc_embedding.weight.detach()))
        x = self.pos(x)
        h = self.plm(x, lens, causal=True)
        logits = ops.linear(h, pack.pack_linear(self.predict_layer.weight))
        return logits, p_codes[:, 1:]

    def infer(self, tc_latent: torch.Tensor, return_logits: bool = False, sampling: S.Sampling = None, keys=None,
              context=None, pinned=None):
        """Greedy AR decode, BOS = vq_bins, exactly T steps, NON-causal full recompute per step
        (models/megatts2.py:165-181).  tc_latent (B,T,tc_dim) -> (B,T) int64 [, (B,T,vq_bins) logits].

        ``sampling`` (opt-in, megatts2_b200.sampling.Sampling): each step's code is drawn on the device instead of the
        argmax, row b keyed by ``keys[b]`` (B 64-bit integers, default arange(B)); the returned logits stay the raw ones.
        The seed and the keys are inputs of the replayed CUDA graph, so a new seed needs no new capture.

        ``context`` (opt-in in-context prompting; a ``PLMContext`` or a list of them, joined in order): the target is
        decoded as the continuation of the context's P rows, as the model was trained: step j sees the latents
        [context; tc_latent[:, :j+1]] at positions 0..P+j and the codes [BOS, context codes, c_0 .. c_{j-1}].  The codes
        and logits are the target's only; a sampled step j draws the noise of ``infer``'s step j.  The context is a graph
        input, so a new context of the same shape needs no new capture.

        ``pinned`` (opt-in code pins, the prosody half of speech editing): (B, T) ints, -1 leaves step j of utterance b
        free and 0..vq_bins-1 fixes its code, which is written into the history in place of the pick, so the free steps
        decode after it (include/megatts2_b200.h, mtts_plm_infer_pinned_f32).  A step pinned in every utterance is never
        enqueued: step j reads the codes of steps < j only, so the free steps run the same kernels on the same data as a
        decode of every step, and an edit costs the free steps alone.  The codes returned hold the pins.  With
        ``return_logits`` every step runs, and a pinned step's logits score its pinned history (teacher forcing).  The pins
        are a graph input; which steps run is part of the graph key, so new pin values with the same free steps replay
        without a new capture.  Combines with ``sampling`` (a pinned row draws nothing; the other rows' draws do not
        change) and ``context``."""
        _eval_only(self)
        tc = _dev_rows(tc_latent, "tc_latent")
        B, T, _ = tc.shape
        pin = None if pinned is None else S.pinned_codes(pinned, B, T, self.vq_bins)
        ctx = _context_inputs(context, B, self.tc_latent_dim, self.vq_bins, tc.device)
        smp = _sampling_inputs(sampling, keys, B, tc.device)
        if pin is not None:
            return self._decode_pinned(tc, smp, ctx, pin.to(tc.device), S.pinned_runs(pin, return_logits),
                                       return_logits)
        return self._decode(tc, 1, None, smp, 0, T, None, return_logits, ctx)

    def _decode_pinned(self, tc, smp, ctx, pin, runs, return_logits):
        """``infer`` with the (B, T) int32 device code pins ``pin``: one graphed call that builds the code state (BOS, the
        context's codes, the pins >= 0) and enqueues mtts_plm_infer_pinned_f32 once per run [j0, j1) of ``runs``, the
        steps with a free row.  -> the state's target columns (B, T) int64 [, logits (B, T, V)]."""
        B, T, V = tc.shape[0], tc.shape[1], self.vq_bins
        P = 0 if ctx is None else ctx[0].shape[1]
        pl = self._plan_get(tc.device, P + T)
        lib = L.lib()
        m = C.byref(pl.struct)

        def run(tc_, pin_, *rest):
            ctx_, rest = (rest[:2], rest[2:]) if ctx is not None else (None, rest)
            state = torch.full((B, P + T + 1), V, dtype=torch.int64, device=tc_.device)     # column 0 = BOS
            if P:
                state[:, 1:P + 1] = ctx_[1]
            target = state[:, P + 1:]
            target.copy_(torch.where(pin_ >= 0, pin_.to(torch.int64), target))
            codes = torch.empty(B, T, dtype=torch.int64, device=tc_.device)
            logits = torch.empty(B, T, V, dtype=torch.float32, device=tc_.device) if return_logits else None
            if runs:
                ws = ops.workspace(lib.mtts_plm_infer_ctx_workspace_bytes(m, B, P, T), tc_.device)
                s = C.byref(smp[0].struct(*rest)) if smp is not None else None
                c_args = _ctx_args(ctx_) if ctx is not None else (None, 0, 0, None, 0, 0)
                for j0, j1 in runs:
                    L.check(lib.mtts_plm_infer_pinned_f32(m, tc_.data_ptr(), tc_.stride(0), tc_.stride(1), B, T, *c_args,
                                                          j0, j1, state.data_ptr(), codes.data_ptr(),
                                                          logits.data_ptr() if return_logits else None, s,
                                                          pin_.data_ptr(), T, ws.data_ptr(), ws.numel(), ops._stream()))
            target = target.contiguous()
            return (target, logits) if return_logits else (target,)

        inputs = (tc, pin) + (tuple(ctx) if ctx is not None else ()) + (smp[1:] if smp is not None else ())
        key = (pl.serial, B, T, runs, bool(return_logits), tc.stride(0), tc.stride(1), ops.launch_policy_now(),
               None if smp is None else smp[0].graph_key(), None if ctx is None else (ctx[0].shape[0], P))
        out = self._graphs("pinned").run(key, inputs, run)
        return out if return_logits else out[0]

    def _decode(self, tc, K, weights, smp, t0, t1, state, return_logits, ctx=None):
        """Steps [t0, t1) of the decode of B utterances from ``tc``, the (K*B, T, tc_dim) stack of K sources mixed by the
        (B, K) device ``weights``, or by the (B, T, K) schedule with one row per step (None: K = 1, the plain decode).  ``smp``: (sampling, seed, keys), or None for greedy.
        ``state`` None: the whole decode (t0 = 0, t1 = T) on the shared workspace; otherwise a range against that (B, T+1)
        code state, on a private workspace since a captured range pins it.  ``ctx``: (tc8 (Bc, P, tc_dim), codes (Bc, P)) of
        a prompt context, or None; the steps stay target steps and the state is then (B, P+T+1).  The enqueues are
        device-only, so the call replays as a CUDA graph from the second time on; ranges keep their graphs in a cache of
        their own, so streaming never evicts the whole decodes'.  -> codes (B, t1 - t0) int64 [, logits (B, t1 - t0, V),
        or (K, B, t1 - t0, V) when mixed]."""
        B, T, V = tc.shape[0] // K, tc.shape[1], self.vq_bins
        mix, ranged = weights is not None, state is not None
        sched = mix and weights.dim() == 3
        P = 0 if ctx is None else ctx[0].shape[1]
        pl = self._plan_get(tc.device, P + T)
        lib = L.lib()
        m = C.byref(pl.struct)
        if ctx is not None:   # so do the context entries
            entry = lib.mtts_plm_infer_ctx_range_f32 if ranged else lib.mtts_plm_infer_ctx_f32
        elif sched:      # the mix entries take the sampling as a nullable argument
            entry = lib.mtts_plm_infer_mix_steps_range_f32 if ranged else lib.mtts_plm_infer_mix_steps_f32
        elif mix:
            entry = lib.mtts_plm_infer_mix_range_f32 if ranged else lib.mtts_plm_infer_mix_f32
        elif smp is None:
            entry = lib.mtts_plm_infer_range_f32 if ranged else lib.mtts_plm_infer_f32
        else:
            entry = lib.mtts_plm_infer_range_sample_f32 if ranged else lib.mtts_plm_infer_sample_f32

        def run(tc_, *rest):
            state_, rest = (rest[0], rest[1:]) if ranged else (None, rest)
            w_, rest = (rest[0], rest[1:]) if mix else (None, rest)
            ctx_, rest = (rest[:2], rest[2:]) if ctx is not None else (None, rest)
            codes = torch.empty(B, T, dtype=torch.int64, device=tc_.device)
            logits = torch.empty(K * B, T, V, dtype=torch.float32, device=tc_.device) if return_logits else None
            nbytes = (lib.mtts_plm_infer_mix_workspace_bytes(m, K, B, T) if mix else
                      lib.mtts_plm_infer_ctx_workspace_bytes(m, B, P, T) if ctx is not None else
                      lib.mtts_plm_infer_workspace_bytes(m, B, T))
            if ranged:
                ws, ws_bytes = torch.empty(nbytes + 256, dtype=torch.uint8, device=tc_.device), nbytes
            else:
                ws = ops.workspace(nbytes, tc_.device)
                ws_bytes = ws.numel()
            lat = (tc_.data_ptr(), tc_.stride(0), tc_.stride(1), B, T)
            steps = (t0, t1, state_.data_ptr()) if ranged else ()
            outs = (codes.data_ptr(), logits.data_ptr() if return_logits else None)
            s = C.byref(smp[0].struct(*rest)) if smp is not None else None
            if ctx is not None:
                args = (m,) + lat + _ctx_args(ctx_) + steps + outs + (s,)
            elif mix:
                w_args = (w_.data_ptr(), T * K, K) if sched else (w_.data_ptr(),)
                args = (m, K) + lat + w_args + steps + outs + (s,)
            else:
                args = (m,) + lat + steps + outs + ((s,) if s is not None else ())
            L.check(entry(*args, ws.data_ptr(), ws_bytes, ops._stream()))
            return (codes[:, t0:t1], logits[:, t0:t1]) if return_logits else (codes[:, t0:t1],)

        inputs = ((tc,) + ((state,) if ranged else ()) + ((weights,) if mix else ()) + (tuple(ctx) if ctx is not None else ())
                  + (smp[1:] if smp is not None else ()))
        key = (pl.serial, K, mix, B, T, t0, t1, bool(return_logits), tc.stride(0), tc.stride(1), ops.launch_policy_now(),
               None if smp is None else smp[0].graph_key(), None if ctx is None else (ctx[0].shape[0], P), sched)
        out = self._graphs("range" if ranged else "main").run(key, inputs, run)
        if not return_logits:
            return out[0]
        return out[0], (out[1].reshape(K, B, t1 - t0, V) if mix else out[1])

    def infer_mix(self, tc_latents, weights, return_logits: bool = False, sampling: S.Sampling = None, keys=None,
                  pinned=None):
        """Prosody interpolation (Mega-TTS 2): the ``infer`` decode of B utterances from a weighted mixture of K sources'
        code distributions.  ``tc_latents``: K tensors (B, T, tc_dim), one per source (e.g. ``tc_latent`` from different
        prosody prompts); ``weights``: (K,) or (B, K), >= 0, each row with a positive sum (normalised per utterance).  All
        sources share one code history; step t picks c_t from l = log sum_k w^_k softmax(logits of source k), greedily or
        by ``sampling`` / ``keys`` as in ``infer``; with exactly one positive weight in a row, l is that source's raw
        logits row (include/megatts2_b200.h states the contract).  -> codes (B, T) int64 [, logits (K, B, T, vq_bins), the
        raw per-source logits].  Replays as a CUDA graph whose inputs are the latents, the weights, the seed and the keys,
        so new weight values need no new capture.

        ``weights`` may also be a schedule (B, T, K): step t of utterance b then mixes by row (b, t), under the same rules
        per row, so the prosody can follow one prompt in one part of the utterance and another elsewhere
        (``ops.mix_step_weights`` makes such a schedule from per-phone weights).  Code pins are not built for the mix."""
        _eval_only(self)
        _no_code_pins(pinned, "infer_mix")
        tc, w = _mix_sources(tc_latents, weights, self.tc_latent_dim, "prosody mix")
        K, (B, T, _) = len(tc_latents), tc_latents[0].shape
        return self._decode(tc, K, w, _sampling_inputs(sampling, keys, B, tc.device), 0, T, None, return_logits)

    def begin_decode(self, tc_latent, sampling: S.Sampling = None, keys=None, weights=None, context=None,
                     pinned=None) -> "PLMDecode":
        """Start a resumable ``infer``: returns the decode state that ``decode_until`` advances.  Decoding through step T in
        any number of ranges gives ``infer``'s codes and logits (same ``sampling``, ``keys`` and ``context``).  With
        ``weights`` ((K,), (B, K) or a (B, T, K) schedule), ``tc_latent`` is the list of K sources of ``infer_mix`` and the
        ranges give ``infer_mix``'s codes and logits (not with a context).  Code pins are ``infer``'s alone."""
        _eval_only(self)
        _no_code_pins(pinned, "begin_decode")
        K, w = 1, None
        if weights is not None:
            if context is not None:
                raise L.MttsError("begin_decode: a context does not combine with prosody mix weights")
            K = len(tc_latent)
            tc, w = _mix_sources(tc_latent, weights, self.tc_latent_dim, "prosody mix")
        else:
            tc = _dev_rows(tc_latent, "tc_latent")
        B, T = tc.shape[0] // K, tc.shape[1]
        ctx = _context_inputs(context, B, self.tc_latent_dim, self.vq_bins, tc.device)
        P = 0 if ctx is None else ctx[0].shape[1]
        state = torch.full((B, P + T + 1), self.vq_bins, dtype=torch.int64, device=tc.device)   # column 0 = BOS
        if P:
            state[:, 1:P + 1] = ctx[1]
        smp = _sampling_inputs(sampling, keys, B, tc.device) or (None, None, None)
        return PLMDecode(tc, state, *smp, w, ctx)

    def decode_until(self, dec: "PLMDecode", t1: int, return_logits: bool = False):
        """Run steps [dec.t, t1) of the decode begun by ``begin_decode`` -> the new codes (B, t1 - dec.t) int64 [, their
        logits (B, t1 - dec.t, vq_bins)].  Each range replays as a CUDA graph keyed by (B, T, t0, t1), from a cache of its
        own (``_graphs("range")``), so streaming never evicts ``infer``'s graphs; a captured range pins a private workspace
        of ``mtts_plm_infer_workspace_bytes(B, T)`` bytes.  A mixed decode (``begin_decode(..., weights=...)``) returns the
        logits as (K, B, t1 - dec.t, vq_bins) and replays with the weights as a graph input."""
        _eval_only(self)
        B, T, t0, t1 = dec.B, dec.T, dec.t, int(t1)
        if not t0 <= t1 <= T:
            raise L.MttsError(f"decode_until: t1 = {t1} outside [{t0}, {T}]")
        if t1 == t0:
            codes = torch.empty(B, 0, dtype=torch.int64, device=dec.tc.device)
            lg_shape = (B, 0, self.vq_bins) if dec.weights is None else (dec.K, B, 0, self.vq_bins)
            return (codes, torch.empty(*lg_shape, device=dec.tc.device)) if return_logits else codes
        smp = None if dec.sampling is None else (dec.sampling, dec.seed, dec.keys)
        out = self._decode(dec.tc, dec.K, dec.weights, smp, t0, t1, dec.state, return_logits, dec.ctx)
        # a replay advanced the graph's copy of the state, not dec.state
        dec.target[:, t0:t1].copy_(out[0] if return_logits else out)
        dec.t = t1
        return out

    def infer_causal(self, tc_latent: torch.Tensor, return_logits: bool = False, sampling: S.Sampling = None,
                     keys=None, context=None, pinned=None):
        """OPT-IN causal KV-cache greedy decode (SURVEY.md 8f-1) - NOT what the reference's ``infer`` computes.

        ``infer`` re-runs the stack bidirectionally every step (models/megatts2.py:177); this decode follows the
        *training* semantics of ``forward`` (causal=True, models/megatts2.py:158): row t attends to rows <= t, so
        each step computes one row per utterance against per-layer K/V caches (O(T) instead of O(T^2)).  Its
        logits equal the teacher-forced ``forward`` logits evaluated on its own output.  Same I/O as ``infer``,
        ``sampling`` and ``keys`` included (the same noise as ``infer`` for a given seed, key and step).

        ``context`` (as in ``infer``): the causal form of the in-context decode.  The context's P rows run through the stack
        once, as one teacher-forced causal pass that fills the K/V caches, then T single-row steps follow; the logits
        equal the teacher-forced ``forward`` over [context; target] at the decoded codes.  Code pins are ``infer``'s
        alone."""
        _eval_only(self)
        _no_code_pins(pinned, "infer_causal")
        tc = _dev_rows(tc_latent, "tc_latent")
        B, T, _ = tc.shape
        ctx = _context_inputs(context, B, self.tc_latent_dim, self.vq_bins, tc.device)
        P = 0 if ctx is None else ctx[0].shape[1]
        pl = self._plan_get(tc.device, P + T)
        lib = L.lib()
        m = C.byref(pl.struct)
        codes = torch.empty(B, T, dtype=torch.int64, device=tc.device)
        logits = torch.empty(B, T, self.vq_bins, dtype=torch.float32, device=tc.device) if return_logits else None
        smp = _sampling_inputs(sampling, keys, B, tc.device)     # held until the call: the struct points into it
        s = None if smp is None else C.byref(sampling.struct(*smp[1:]))
        lat = (tc.data_ptr(), tc.stride(0), tc.stride(1), B, T)
        outs = (codes.data_ptr(), logits.data_ptr() if return_logits else None)
        if ctx is not None:
            ws = ops.workspace(lib.mtts_plm_decode_causal_ctx_workspace_bytes(m, B, P, T), tc.device)
            L.check(lib.mtts_plm_decode_causal_ctx_f32(m, *lat, *_ctx_args(ctx), *outs, s, ws.data_ptr(), ws.numel(),
                                                       ops._stream()))
            return (codes, logits) if return_logits else codes
        ws = ops.workspace(lib.mtts_plm_decode_causal_workspace_bytes(m, B, T), tc.device)
        entry = lib.mtts_plm_decode_causal_f32 if smp is None else lib.mtts_plm_decode_causal_sample_f32
        L.check(entry(m, *lat, *outs, *(() if s is None else (s,)), ws.data_ptr(), ws.numel(), ops._stream()))
        return (codes, logits) if return_logits else codes

    @classmethod
    def from_pretrained(cls, ckpt: str, config: str) -> "MegaPLM":
        with open(config, "r") as f:
            plm = instantiate_class(args=(), init=yaml.safe_load(f)['model']['plm'])
        sd = {k[4:]: v for k, v in torch.load(ckpt, map_location="cpu")['state_dict'].items() if k.startswith('plm.')}
        plm.load_state_dict(sd, strict=True)
        return plm


class PLMDecode:
    """State of one resumable PLM decode (``MegaPLM.begin_decode``): the latent ``tc`` (B, T, tc_dim), the code state
    (B, P+T+1) int64 (column 0 = BOS, columns 1..P the context's codes, column P+1+t the code of target step t once
    decoded), the sampling parameters with the seed and row keys as device tensors (None for greedy), and ``t``, the number
    of target steps decoded.  A mixed decode also holds the (B, K) device ``weights``, and ``tc`` is then the (K*B, T,
    tc_dim) stack of its K sources (or the (B, T, K) schedule); a decode with a context holds ``ctx`` = (tc8 (Bc, P, tc_dim), codes (Bc, P)) and P."""

    def __init__(self, tc, state, sampling, seed, keys, weights=None, ctx=None):
        self.tc, self.state, self.sampling, self.seed, self.keys = tc, state, sampling, seed, keys
        self.weights, self.ctx = weights, ctx
        self.K = 1 if weights is None else weights.shape[-1]
        self.P = 0 if ctx is None else ctx[0].shape[1]
        self.B, self.T = state.shape[0], tc.shape[1]
        self.t = 0

    @property
    def target(self):
        """The target's code columns of the state, (B, T) (a view; columns >= t are not decoded yet)."""
        return self.state[:, self.P + 1:]

    @property
    def codes(self):
        """The codes decoded so far, (B, t) (a view of the state)."""
        return self.target[:, :self.t]


class MegaADM(pack.PlanMixin, nn.Module):
    def __init__(self, n_layers: int = 8, n_heads: int = 8, emb_dim: int = 256, tc_latent_dim: int = 512,
                 tc_emb_dim: int = 256, dropout: float = 0.1, max_duration_token: int = 256):
        super().__init__()
        d_model = emb_dim + tc_emb_dim
        self.adm = TransformerEncoder(
            TransformerEncoderLayer(dim=d_model, ff_dim=emb_dim * 4, n_heads=n_heads, dropout=dropout, conv_ff=False),
            num_layers=n_layers)
        self.dt_linear_emb = nn.Linear(1, emb_dim, bias=False)
        self.tc_linear_emb = nn.Linear(tc_latent_dim, tc_emb_dim, bias=False)
        self.pos_emb = SinePositionalEmbedding(d_model)
        self.predict_layer = nn.Linear(d_model, 1, bias=False)
        self.max_duration_token = max_duration_token
        self.emb_dim, self.tc_latent_dim, self.tc_emb_dim = emb_dim, tc_latent_dim, tc_emb_dim
        self._plan = None

    def _plan_get(self, device, T):
        def fill(pl, s):
            s.w_dt = pl.p(self.dt_linear_emb.weight.detach()[:, 0].contiguous())
            s.w_tc = pl.p(pack.pack_linear(self.tc_linear_emb.weight))
            s.w_predict = pl.p(self.predict_layer.weight.detach()[0].contiguous())
            s.emb_dim, s.tc_dim, s.tc_emb_dim = self.emb_dim, self.tc_latent_dim, self.tc_emb_dim
        return _ar_plan(self, self.adm, self.pos_emb, L.ADM, device, T, fill)

    def forward(self, tc_latents: torch.Tensor, duration_tokens: torch.Tensor, lens: torch.Tensor):
        """Teacher-forced duration regression (models/megatts2.py:233-255); training mode runs on autograd Functions."""
        if self.training:
            dt_emb = A.linear(duration_tokens[:, :-1].float(), self.dt_linear_emb.weight, None)
            tc_emb = A.linear(tc_latents, self.tc_linear_emb.weight, None)
            x = self.pos_emb(torch.cat([tc_emb, dt_emb], dim=-1))
            h = self.adm(x, lens, causal=True)
            return A.linear(h, self.predict_layer.weight, None)[..., 0], duration_tokens[:, 1:, 0]
        B, T, _ = tc_latents.shape
        dev = tc_latents.device
        x = torch.empty(B, T, self.tc_emb_dim + self.emb_dim, dtype=torch.float32, device=dev)
        x[..., :self.tc_emb_dim].copy_(ops.linear(tc_latents, pack.pack_linear(self.tc_linear_emb.weight)))
        x[..., self.tc_emb_dim:].copy_(ops.linear(duration_tokens[:, :-1].contiguous().float(),
                                                  pack.pack_linear(self.dt_linear_emb.weight)))
        x = self.pos_emb(x)
        h = self.adm(x, lens, causal=True)
        pred = ops.linear(h, pack.pack_linear(self.predict_layer.weight))[..., 0]
        return pred, duration_tokens[:, 1:, 0]

    def infer(self, tc_latents: torch.Tensor, return_raw: bool = False, pinned=None):
        """AR duration regression, raw float feedback, non-causal full recompute, final
        (p + 0.5) -> int32 -> clamp(1, 128)  (models/megatts2.py:257-275).
        tc_latents (B,T,512) -> (B,T,1) int32 [, raw (B,T) fp32].

        ``pinned`` (B, T) ints, -1 free or 1..127 frames: a pinned phone's value is fed back into the loop in place of
        the prediction, so the later phones are decoded after it, and it comes out exactly as pinned (raw holds it too;
        include/megatts2_b200.h, mtts_adm_infer_pinned_f32).  The pins are an input of the replayed CUDA graph."""
        _eval_only(self)
        tc = _dev_rows(tc_latents, "tc_latents")
        B, T, _ = tc.shape
        pin = None if pinned is None else S.pinned_durations(pinned, B, T).to(tc.device)
        pl = self._plan_get(tc.device, T)
        lib = L.lib()

        def run(tc_, *pin_):
            dur = torch.empty(B, T, dtype=torch.int32, device=tc_.device)
            raw = torch.empty(B, T, dtype=torch.float32, device=tc_.device) if return_raw else None
            outs = (dur.data_ptr(), raw.data_ptr() if return_raw else None)
            if pin_:
                ws = ops.workspace(lib.mtts_adm_infer_mix_workspace_bytes(C.byref(pl.struct), 1, B, T), tc_.device)
                L.check(lib.mtts_adm_infer_pinned_f32(C.byref(pl.struct), 1, tc_.data_ptr(), tc_.stride(0),
                                                      tc_.stride(1), B, T, None, 0, 0, *outs, None, pin_[0].data_ptr(),
                                                      T, ws.data_ptr(), ws.numel(), ops._stream()))
                return (dur, raw) if return_raw else (dur,)
            ws = ops.workspace(lib.mtts_adm_infer_workspace_bytes(C.byref(pl.struct), B, T), tc_.device)
            L.check(lib.mtts_adm_infer_f32(C.byref(pl.struct), tc_.data_ptr(), tc_.stride(0), tc_.stride(1), B, T,
                                           *outs, ws.data_ptr(), ws.numel(), ops._stream()))
            return (dur, raw) if return_raw else (dur,)

        out = self._graphs().run(("adm", pl.serial, B, T, bool(return_raw), tc.stride(0), tc.stride(1),
                                  ops.launch_policy_now(), pin is not None), (tc,) if pin is None else (tc, pin), run)
        dur = out[0]
        raw = out[1] if return_raw else None
        dur = dur.unsqueeze(-1)
        return (dur, raw) if return_raw else dur

    def infer_mix(self, tc_latents, weights, return_raw: bool = False, pinned=None):
        """Duration interpolation: the ``infer`` decode of B utterances from a weighted mean of K sources' duration
        predictions.  ``tc_latents``: K tensors (B, T, tc_dim), one per source (e.g. ``tc_latent`` of different prompts);
        ``weights``: (K,) or (B, K), >= 0, each row with a positive sum (normalised per utterance).  All sources share one
        raw-duration history; step t runs every source's ``infer`` step and feeds back r = sum_k w^_k y_k, the weighted
        mean of their readouts; with exactly one positive weight in a row, r is that source's readout bit for bit
        (include/megatts2_b200.h states the contract).  -> durations (B, T, 1) int32 [, raw (B, T) fp32 (the mixed values),
        raw_src (K, B, T) fp32 (every source's readout)].  Replays as a CUDA graph whose inputs are the latents and the
        weights, so new weight values need no new capture.

        ``weights`` may also be a schedule (B, T, K), one row per phone: step t, the duration of phone t, mixes by row
        (b, t).  ``pinned`` (B, T) as in ``infer``: a pinned phone feeds back its pin in place of the mixed value (raw_src
        keeps every source's own readout)."""
        _eval_only(self)
        tc, w = _mix_sources(tc_latents, weights, self.tc_latent_dim, "duration mix")
        K, (B, T, _) = len(tc_latents), tc_latents[0].shape
        sched = w.dim() == 3
        pin = None if pinned is None else S.pinned_durations(pinned, B, T).to(tc.device)
        pl = self._plan_get(tc.device, T)
        lib = L.lib()

        def run(tc_, w_, *pin_):
            dur = torch.empty(B, T, dtype=torch.int32, device=tc_.device)
            raw = torch.empty(B, T, dtype=torch.float32, device=tc_.device) if return_raw else None
            raw_src = torch.empty(K, B, T, dtype=torch.float32, device=tc_.device) if return_raw else None
            ws = ops.workspace(lib.mtts_adm_infer_mix_workspace_bytes(C.byref(pl.struct), K, B, T), tc_.device)
            lat = (C.byref(pl.struct), K, tc_.data_ptr(), tc_.stride(0), tc_.stride(1), B, T)
            outs = (dur.data_ptr(), raw.data_ptr() if return_raw else None, raw_src.data_ptr() if return_raw else None,
                    ws.data_ptr(), ws.numel(), ops._stream())
            if pin_:
                L.check(lib.mtts_adm_infer_pinned_f32(*lat, w_.data_ptr(), *((T * K, K) if sched else (K, 0)),
                                                      *outs[:3], pin_[0].data_ptr(), T, *outs[3:]))
            elif sched:
                L.check(lib.mtts_adm_infer_mix_steps_f32(*lat, w_.data_ptr(), T * K, K, *outs))
            else:
                L.check(lib.mtts_adm_infer_mix_f32(*lat, w_.data_ptr(), *outs))
            return (dur, raw, raw_src) if return_raw else (dur,)

        out = self._graphs().run(("adm_mix", pl.serial, K, B, T, bool(return_raw), tc.stride(0), tc.stride(1),
                                  ops.launch_policy_now(), sched, pin is not None),
                                 (tc, w) if pin is None else (tc, w, pin), run)
        dur = out[0].unsqueeze(-1)
        return (dur, out[1], out[2]) if return_raw else dur

    def infer_causal(self, tc_latents: torch.Tensor, return_raw: bool = False):
        """OPT-IN causal KV-cache duration decode (SURVEY.md 8f-1) - NOT what the reference's ``infer`` computes:
        the training semantics of ``forward`` (causal=True, models/megatts2.py:244) with ``infer``'s raw-float
        feedback and final rounding; one row per utterance per step against K/V caches.  Same I/O as ``infer``."""
        _eval_only(self)
        tc = _dev_rows(tc_latents, "tc_latents")
        B, T, _ = tc.shape
        pl = self._plan_get(tc.device, T)
        lib = L.lib()
        dur = torch.empty(B, T, dtype=torch.int32, device=tc.device)
        raw = torch.empty(B, T, dtype=torch.float32, device=tc.device) if return_raw else None
        ws = ops.workspace(lib.mtts_adm_decode_causal_workspace_bytes(C.byref(pl.struct), B, T), tc.device)
        L.check(lib.mtts_adm_decode_causal_f32(C.byref(pl.struct), tc.data_ptr(), tc.stride(0), tc.stride(1), B, T,
                                               dur.data_ptr(), raw.data_ptr() if return_raw else None,
                                               ws.data_ptr(), ws.numel(), ops._stream()))
        dur = dur.unsqueeze(-1)
        return (dur, raw) if return_raw else dur

    @classmethod
    def from_pretrained(cls, ckpt: str, config: str) -> "MegaADM":
        with open(config, "r") as f:
            adm = instantiate_class(args=(), init=yaml.safe_load(f)['model']['adm'])
        sd = {k[4:]: v for k, v in torch.load(ckpt, map_location="cpu")['state_dict'].items() if k.startswith('adm.')}
        adm.load_state_dict(sd, strict=True)
        return adm


# ------------------------------------------------------------------------------------------
# Overlapped prompt re-vocode (Megatts._synthesize): defaults of MEGATTS2_REVOCODE_SMS / _FRAC / _FROM
REVOCODE_SMS_DEFAULT = 0
REVOCODE_FRAC_DEFAULT = 1.0
REVOCODE_FROM_DEFAULT = "mrte"

HIFIGAN_V1 = dict(in_channels=80, upsample_initial_channel=512, upsample_factors=(8, 8, 2, 2),
                  upsample_kernel_sizes=(16, 16, 4, 4), resblock_kernel_sizes=(3, 7, 11),
                  resblock_dilation_sizes=((1, 3, 5), (1, 3, 5), (1, 3, 5)), inference_padding=5)


class HifiganGenerator(pack.PlanMixin, nn.Module):
    """HiFi-GAN V1 generator, weight-norm already folded (speechbrain HifiganGenerator [published
    architecture]; SURVEY.md §2.4 K13 / §8c).  Parameter names: ``conv_pre.{weight,bias}``,
    ``ups.{i}.{weight,bias}`` (ConvTranspose1d layout (Cin, Cout, k)),
    ``resblocks.{n}.convs{1,2}.{m}.{weight,bias}``, ``conv_post.{weight,bias}``."""

    def __init__(self, **cfg):
        super().__init__()
        c = dict(HIFIGAN_V1)
        c.update(cfg)
        self.cfg = c
        ch = c["upsample_initial_channel"]
        self.conv_pre = nn.Conv1d(c["in_channels"], ch, 7)
        self.ups = nn.ModuleList()
        self.resblocks = nn.ModuleList()
        for i, (u, k) in enumerate(zip(c["upsample_factors"], c["upsample_kernel_sizes"])):
            co = ch // (2 ** (i + 1))
            self.ups.append(nn.ConvTranspose1d(ch // (2 ** i), co, k, stride=u, padding=(k - u) // 2))
            for j, rk in enumerate(c["resblock_kernel_sizes"]):
                rb = nn.Module()
                rb.convs1 = nn.ModuleList([nn.Conv1d(co, co, rk, dilation=d) for d in c["resblock_dilation_sizes"][j]])
                rb.convs2 = nn.ModuleList([nn.Conv1d(co, co, rk) for _ in c["resblock_dilation_sizes"][j]])
                self.resblocks.append(rb)
        self.conv_post = nn.Conv1d(ch // (2 ** len(c["upsample_factors"])), 1, 7)
        self._plan = None

    def _plan_get(self):
        engine = getattr(self, "engine", None)
        engine = pack.default_engine() if engine is None else int(engine)
        sig = pack.signature(list(self.parameters())) + (engine,)
        if self._plan is None or self._plan.sig != sig:
            c = self.cfg
            pl = pack.Plan()
            pl.sig = sig
            s = L.Hifigan()
            s.engine = engine
            fmt = pack.engine_fmt(engine)
            s.in_channels, s.ch0 = c["in_channels"], c["upsample_initial_channel"]
            s.n_ups, s.n_kernels = len(c["upsample_factors"]), len(c["resblock_kernel_sizes"])
            s.inference_padding = c["inference_padding"]
            s.w_pre, s.b_pre = pl.p(pack.pack_conv(self.conv_pre.weight)), pl.p(self.conv_pre.bias)
            for i, (u, k) in enumerate(zip(c["upsample_factors"], c["upsample_kernel_sizes"])):
                s.up_factor[i], s.up_kernel[i] = u, k
                wp, bp = pack.pack_conv_transpose(self.ups[i].weight, self.ups[i].bias, u)
                s.w_up[i], s.b_up[i] = pl.p(wp), pl.p(bp)
                if engine >= 1:     # (2, Cin, s*Cout) fp32 -> (3 | 2 | 1, 2, s*Cout, Cin) operand planes
                    tup = pack.pack_conv_transpose_tc_planes(wp, fmt)
                    pl.keep.append(tup)
                    s.w_up_tc[i] = tup.data_ptr()
            arr = (L.HifiganResblock * len(self.resblocks))()
            for n, rb in enumerate(self.resblocks):
                j = n % s.n_kernels
                arr[n].k = c["resblock_kernel_sizes"][j]
                assert len(rb.convs1) == 3
                for m in range(3):
                    arr[n].dil[m] = c["resblock_dilation_sizes"][j][m]
                    arr[n].w1[m], arr[n].b1[m] = pl.p(pack.pack_conv(rb.convs1[m].weight)), pl.p(rb.convs1[m].bias)
                    arr[n].w2[m], arr[n].b2[m] = pl.p(pack.pack_conv(rb.convs2[m].weight)), pl.p(rb.convs2[m].bias)
                    if engine >= 1:
                        t1, t2 = pack.pack_conv_tc_planes(rb.convs1[m].weight, fmt), pack.pack_conv_tc_planes(rb.convs2[m].weight, fmt)
                        pl.keep += [t1, t2]
                        arr[n].w1_tc[m], arr[n].w2_tc[m] = t1.data_ptr(), t2.data_ptr()
            pl.hold(arr)
            s.resblocks = C.cast(arr, C.POINTER(L.HifiganResblock))
            s.w_post, s.b_post = pl.p(pack.pack_conv(self.conv_post.weight)), pl.p(self.conv_post.bias)
            pl.struct = s
            self._plan = pl
        return self._plan

    def receptive_field(self) -> int:
        """Half-width in mel frames of what one output sample depends on, rounded up: conv_pre, then per stage the
        transposed conv's reach and the widest ResBlock (two convs per dilation), and conv_post, each converted from
        samples at that stage's rate to frames.  A window of mel frames vocoded on its own gives the whole sequence's
        samples for the frames at least this far from each window edge that is not a sequence edge."""
        from fractions import Fraction
        c = self.cfg
        r = Fraction((self.conv_pre.kernel_size[0] - 1) // 2)
        rate = 1                                                  # samples per mel frame at the current stage
        for u, k in zip(c["upsample_factors"], c["upsample_kernel_sizes"]):
            r += Fraction(k - 1 - (k - u) // 2, u * rate)         # output j reads inputs down to (j + pad - k + 1) / u
            rate *= u
            r += Fraction(max(sum((rk - 1) // 2 * (d + 1) for d in dils)
                              for rk, dils in zip(c["resblock_kernel_sizes"], c["resblock_dilation_sizes"])), rate)
        r += Fraction((self.conv_post.kernel_size[0] - 1) // 2, rate)
        return math.ceil(r)

    def out_len(self, T):
        n = T + 2 * self.cfg["inference_padding"]
        for u in self.cfg["upsample_factors"]:
            n *= u
        return n

    def inference_cl(self, mel_cl: torch.Tensor) -> torch.Tensor:
        """mel (B, T, 80) channels-last -> wav (B, 1, 256*(T+10))."""
        mel = _dev_rows(mel_cl, "mel")
        B, T, _ = mel.shape
        pl = self._plan_get()
        lib = L.lib()
        wav = torch.empty(B, 1, self.out_len(T), dtype=torch.float32, device=mel.device)
        ws = ops.workspace(lib.mtts_hifigan_workspace_bytes(C.byref(pl.struct), B, T), mel.device)
        L.check(lib.mtts_hifigan_forward_f32(C.byref(pl.struct), mel.data_ptr(), mel.stride(0), mel.stride(1), B, T,
                                             wav.data_ptr(), wav.stride(0), ws.data_ptr(), ws.numel(), ops._stream()))
        return wav

    def inference(self, c: torch.Tensor, padding: bool = True) -> torch.Tensor:
        """c (B, 80, T) -> (B, 1, 256*(T+10))"""
        assert padding, "inference without padding is not on the synthesis path"
        return self.inference_cl(ops.to_channels_last(c))


def convert_speechbrain_hifigan_state_dict(sd):
    """speechbrain ``HifiganGenerator`` checkpoint keys -> this module's keys, folding weight norm.

    speechbrain wraps every conv as ``<name>.conv`` and applies ``torch.nn.utils.weight_norm`` (dim 0), so a
    ``generator.ckpt`` holds ``conv_pre.conv.weight_g / weight_v / bias``, ``ups.{i}.conv.*``,
    ``resblocks.{n}.convs{1,2}.{m}.conv.*``, ``conv_post.conv.*`` (or, with the parametrization API,
    ``...conv.parametrizations.weight.original0 / original1``) [published layout, restated from memory: speechbrain is
    not vendored by the reference - SURVEY.md 8c].  Folded weight: ``w = g * v / ||v||`` with the norm over every dim but 0
    (what ``remove_weight_norm`` leaves behind, which ``HIFIGAN.decode_batch`` calls before its first inference).  Keys
    that are already in this module's layout pass through."""
    out, groups = {}, {}
    for k, v in sd.items():
        k2 = k[len("generator."):] if k.startswith("generator.") else k
        k2 = k2.replace(".conv.", ".")
        for a, b in ((".parametrizations.weight.original0", ".weight_g"), (".parametrizations.weight.original1", ".weight_v")):
            k2 = k2.replace(a, b)
        if k2.endswith(".weight_g") or k2.endswith(".weight_v"):
            groups.setdefault(k2[:-9], {})[k2[-1]] = v
        else:
            out[k2] = v
    for base, gv in groups.items():
        if set(gv) != {"g", "v"}:
            raise L.MttsError(f"weight-norm pair incomplete for {base!r}")
        v = gv["v"].float()
        norm = v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (v.dim() - 1)))
        out[base + ".weight"] = gv["g"].float().reshape_as(norm) * v / norm
    return out


class HIFIGAN(nn.Module):
    """speechbrain.pretrained.HIFIGAN call surface used by the reference
    (models/megatts2.py:321-323, 370-372): ``from_hparams(source=...)``, ``eval()``,
    ``decode_batch(mel (B,80,T)) -> (B,1,samples)``.  There is no network here: ``source`` must be a local
    directory holding ``generator.ckpt`` (the file speechbrain's hyperparams.yaml names) or a checkpoint file, or an
    explicit ``state_dict`` must be given; anything else raises instead of silently returning a randomly
    initialised vocoder."""

    def __init__(self, generator: HifiganGenerator = None):
        super().__init__()
        self.generator = generator if generator is not None else HifiganGenerator()

    @classmethod
    def from_hparams(cls, source=None, state_dict=None, device=None, random_init=False, **kw):
        import os
        m = cls()
        if state_dict is None and source is not None:
            path = os.path.join(source, "generator.ckpt") if os.path.isdir(source) else source
            if os.path.isfile(path):
                state_dict = torch.load(path, map_location="cpu")
                if isinstance(state_dict, dict) and "state_dict" in state_dict:
                    state_dict = state_dict["state_dict"]
        if state_dict is not None:
            m.generator.load_state_dict(convert_speechbrain_hifigan_state_dict(state_dict), strict=True)
        elif not random_init:
            raise L.MttsError(
                f"HIFIGAN.from_hparams(source={source!r}): no local generator checkpoint found and no state_dict given "
                "(this build cannot download speechbrain/tts-hifigan-libritts-16kHz); pass source=<dir with generator.ckpt>, "
                "state_dict=..., or random_init=True for synthetic-weight benchmarks")
        if device is not None:
            m = m.to(device)
        return m.eval()

    def decode_batch(self, spectrogram: torch.Tensor, mel_lens=None, hop_len=None) -> torch.Tensor:
        """mel (B,80,T) -> (B,1,256*(T+10)).  With ``mel_lens`` and ``hop_len`` the samples past
        ``mel_lens[b] * hop_len`` are zeroed, like speechbrain's ``mask_noise`` [memory]."""
        dev = next(self.generator.parameters()).device
        wav = self.generator.inference(spectrogram.to(dev))
        if (mel_lens is None) != (hop_len is None):
            raise L.MttsError("decode_batch: give both mel_lens and hop_len, or neither")
        if mel_lens is not None:
            keep = (torch.as_tensor(mel_lens).to(torch.int64) * int(hop_len)).to(device=dev, dtype=torch.int32)
            ops.mask_tail(wav, keep)
        return wav

    def decode_batch_cl(self, mel_cl: torch.Tensor) -> torch.Tensor:
        return self.generator.inference_cl(mel_cl)


class _RangeRestart(Exception):
    """An fp16 range flag raised before a stream yielded its first synthesized chunk."""


def _fp16_operands():
    """Whether the default engine feeds the tensor cores fp16 operands (f16x2 or f16), whose range the flag read by
    ``ops.tc_overflow`` guards."""
    return pack.default_engine() in (pack.ENGINE_F16X2, pack.ENGINE_F16)


def _warn_fp16_range(then):
    import warnings
    warnings.warn("megatts2_b200: an activation left the fp16 range of the fp16 operand split; " + then, stacklevel=2)


def _duration_control(phone_tokens, forced_durations, causal_decode, duration_scale, total_frames, pinned_durations):
    """The validated (scale, total, pins) CPU tensors of a synthesis call's duration control, or None without any."""
    if duration_scale is None and total_frames is None and pinned_durations is None:
        return None
    if forced_durations is not None:
        raise L.MttsError("forced_durations replace the ADM's durations; they do not combine with duration_scale, "
                          "total_frames or pinned_durations")
    if pinned_durations is not None and causal_decode:
        raise L.MttsError("pinned_durations run inside the reference-faithful ADM loop, not with causal_decode=True")
    B, Tp = phone_tokens.shape
    return S.duration_control(duration_scale, total_frames, pinned_durations, B, Tp)


class Megatts(nn.Module):
    """Inference orchestrator (models/megatts2.py:295-375).  ``synthesize`` is the tensor-level
    body of the reference's ``forward`` for a batch; ``forward(wavs_dir, text)`` keeps the
    reference signature and needs the reference's host-side text/audio front end
    (librosa, G2P, symbol table - out of the hot path) to be importable."""

    def __init__(self, g_ckpt: str = None, g_config: str = None, plm_ckpt: str = None, plm_config: str = None,
                 adm_ckpt: str = None, adm_config: str = None, symbol_table: str = None, *,
                 generator: MegaG = None, plm: MegaPLM = None, adm: MegaADM = None, hifi_gan: HIFIGAN = None,
                 device="cuda"):
        super().__init__()
        self.generator = generator if generator is not None else MegaG.from_pretrained(g_ckpt, g_config)
        self.plm = plm if plm is not None else MegaPLM.from_pretrained(plm_ckpt, plm_config)
        self.adm = adm if adm is not None else MegaADM.from_pretrained(adm_ckpt, adm_config)
        self.lr = LengthRegulator(HIFIGAN_HOP_LENGTH, 16000, (HIFIGAN_HOP_LENGTH / HIFIGAN_SR * 1000))
        self.hifi_gan = hifi_gan if hifi_gan is not None else HIFIGAN.from_hparams(
            source="speechbrain/tts-hifigan-libritts-16kHz")
        self.symbol_table = symbol_table
        self.to(device)
        self.eval()

    @torch.no_grad()
    def synthesize(self, phone_tokens: torch.Tensor, mels: torch.Tensor, forced_durations: torch.Tensor = None,
                   return_intermediates: bool = False, causal_decode: bool = False, prompt_mels: torch.Tensor = None,
                   return_lengths: bool = False, check_range: bool = True, overlap_prompt: bool = None,
                   sampling: S.Sampling = None, keys=None, prosody_mels=None, prosody_weights=None,
                   duration_weights=None, plm_context=None, duration_scale=None, total_frames=None,
                   pinned_durations=None, timbre_mels=None, timbre_weights=None):
        """phone_tokens (B,Tp) int64, mels (B,Tm,80) prompt mel (frames-major) -> wav (B,1,256*(max sum d + 10)).
        Steps = models/megatts2.py:354-373; every utterance's result equals the reference's batch-1 run on it
        (utterances are independent; the only cross-utterance coupling would be the zero rows the LengthRegulator
        appends to shorter utterances, which the mel decoder and the vocoder must not see - so those two stages run
        per group of equal sum(d), each group one launch sequence, results scattered back; with equal totals - the
        benchmark's forced durations - that is a single group).  All utterances of a call share Tp and Tm (tensors are
        rectangular; ``synthesize_many`` buckets ragged inputs).

        ``forced_durations`` (B,Tp) int32 replaces the ADM output for shape control (the ADM still runs).
        ``prompt_mels`` (B,Tq,80): re-vocode the prompt and prepend it, as the reference does (:371-373).
        ``return_lengths``: also return the valid sample count per utterance (prompt part included).
        ``causal_decode=True`` swaps both AR loops for the opt-in causal KV-cache decode (training semantics; NOT the
        reference's infer() - different ids; SURVEY.md 8f-1).
        ``overlap_prompt``: the prompt re-vocode runs on a side stream with an SM budget (MEGATTS2_REVOCODE_SMS) beside the
        MRTE + ADM stages, which get the remaining SMs (see ``_synthesize``); False forces the sequential form, True the
        overlapped one even when the budget's default is 0.  Waveforms are identical either way (the vocoder has no
        batch- or grid-dependent reduction order); the ADM / MRTE dense layers pick their K split from the SM budget, so
        their fp32 results move within rounding noise.
        ``check_range``: with an fp16 operand engine (f16x2, or the half-precision f16) as the default engine, read the
        range flag after the batch (one 4-byte readback) and, if any activation left the fp16 range, redo the batch on the
        bf16x3 engine.  The check keys off the default engine (``MEGATTS2_ENGINE`` / ``pack.engine_scope``): a module
        whose ``.engine`` is set by hand - e.g. only the vocoder on f16 (``hifi_gan.generator.engine =
        pack.ENGINE_F16``) - is not guarded by it.
        ``sampling`` (opt-in, megatts2_b200.sampling.Sampling): the prosody codes are sampled instead of decoded greedily
        (``MegaPLM.infer``), utterance b keyed by ``keys[b]`` (default arange(B)); the ADM durations stay deterministic.
        The bf16x3 rerun above draws with the same seed and keys.
        ``prosody_mels`` (opt-in prosody interpolation): a list of (B, Tm_k, 80) prosody prompts, with ``prosody_weights``
        (K,) or (B, K), K = 1 + len(prosody_mels); weight 0 belongs to ``mels``.  ``prosody_weights`` may also be
        (B, Tp, K), one row per phone: PLM step t then mixes by the row of the phone owning most of its 8 mel frames
        (``ops.mix_step_weights``, with the durations used), so the prosody changes along the utterance in 8-frame
        steps; ``return_intermediates`` then adds ``prosody_step_weights`` (B, T, K).  Each prompt gives a source latent
        ``mrte.tc_latent(phone_tokens, prompt)``, length-regulated and max-pooled with the target's durations, and the
        codes come from ``MegaPLM.infer_mix`` over the K sources.  The durations (unless ``duration_weights`` is given),
        the mel decoder and the vocoder keep the target's (``mels``) latent, so the timbre stays the target's (``timbre_mels``
        blends it).  Not with
        ``causal_decode``.
        ``duration_weights`` (opt-in duration interpolation, with ``prosody_mels``): (K,) or (B, K), or (B, Tp, K) with one
        row per phone (the ADM's step t is phone t), the same K; weight 0 belongs to ``mels``.  The durations then come from ``MegaADM.infer_mix`` over [the target's latent, *the prompts'
        latents] instead of ``MegaADM.infer`` on the target's alone, so the rhythm moves toward the prompts as well; each
        prompt's latent is computed once and serves both mixes.  ``forced_durations`` still override them.
        ``plm_context`` (opt-in in-context prompting): a ``PLMContext`` (or a list of them, joined in order), e.g. from
        ``generator.plm_context`` on same-speaker prompt utterances; the prosody codes come from ``MegaPLM.infer`` (or
        ``infer_causal`` with ``causal_decode``) with ``context=plm_context``, so the target continues the prompts'
        prosody as in training.  The durations, the mel decoder and the vocoder see the target only.  Not with
        ``prosody_mels``.
        Duration control (opt-in; none of it with ``forced_durations``; include/megatts2_b200.h states the rules):
        ``duration_scale``: a number, (B,) or (B, Tp), finite and > 0, multiplies the ADM's raw durations (above 1 is
        slower); ``total_frames`` (B,) ints: utterance b gets exactly that many mel frames (``wav_lens`` = 256 (L_b + 10)),
        the phones sharing them in proportion to their (scaled) predictions; ``pinned_durations`` (B, Tp) ints, -1 free
        or 1..127: those phones get exactly that many frames, fed back inside the ADM loop so the rest of the utterance
        follows from them (not with ``causal_decode``).  They combine with each other and with ``duration_weights``;
        ``return_intermediates["dt"]`` holds the durations used (``ops.fit_durations`` of the ADM's raw values when a
        scale or a total is given).
        ``timbre_mels`` (opt-in timbre interpolation): a list of (B, Tm_k, 80) timbre prompts, with ``timbre_weights``
        (K,), (B, K) or (B, Tp, K) with one row per phone, K = 1 + len(timbre_mels) <= 8; weight 0 belongs to ``mels``.
        The mel decoder then reads ``MRTE.tc_latent_mix(phone_tokens, [mels, *timbre_mels], timbre_weights)``,
        length-regulated with the durations used, instead of the target's latent, so the voice moves toward the prompts
        (per phone, with a schedule).  The ADM and the prosody LM keep the target's latent (``duration_weights`` and
        ``prosody_weights`` are their controls), so ``tc_latent``, ``dt`` and ``p_codes`` do not change; a full voice blend
        passes the same prompts and weights to all three.  A prompt passed as the same tensor in ``prosody_mels`` and
        ``timbre_mels`` is encoded once, and MRTE's phone encoder runs once per call.  ``return_intermediates`` adds
        ``timbre_latent`` (B, Tp, H).
        All arguments are checked on the host before any device work."""
        dev = phone_tokens.device
        self._check_prosody(phone_tokens, prosody_mels, prosody_weights, causal_decode, duration_weights, plm_context)
        control = _duration_control(phone_tokens, forced_durations, causal_decode, duration_scale, total_frames,
                                    pinned_durations)
        timbre = self._check_timbre(phone_tokens, timbre_mels, timbre_weights)
        args = (phone_tokens, mels, forced_durations, causal_decode, prompt_mels, overlap_prompt, sampling, keys,
                prosody_mels, prosody_weights, duration_weights, plm_context, control)
        out = self._synthesize(*args, timbre=timbre)
        if check_range and _fp16_operands() and ops.tc_overflow(dev):
            _warn_fp16_range("re-running this batch on the bf16x3 engine")
            with pack.engine_scope(pack.ENGINE_BF16X3):
                out = self._synthesize(*args, timbre=timbre)
        if return_intermediates:
            return out
        return (out["wav"], out["wav_lens"]) if return_lengths else out["wav"]

    @torch.no_grad()
    def edit(self, phone_tokens: torch.Tensor, mels: torch.Tensor, orig_phone, orig_durations, orig_codes, span,
             span_frames=None, duration_scale=None, sampling: S.Sampling = None, keys=None, plm_context=None,
             check_range: bool = True, return_lengths: bool = False, return_intermediates: bool = False, **rejected):
        """Speech editing: regenerate the phones [a, b) = ``span[r]`` of an utterance while the durations and prosody
        codes around them stay as they were.  ``orig_phone`` / ``orig_durations`` (B, Tp_o) and ``orig_codes``
        (B, >= ceil(N_o / 8)), N_o the original's frame count, describe the original: ``dt`` and ``p_codes`` of an
        earlier ``synthesize(..., return_intermediates=True)``, or for a recording its aligner durations and the codes of
        its mel (``generator.vqpe(mel)[3][0]``).  ``phone_tokens`` (B, Tp_e) is the edited sentence: row r is
        ``orig_phone[r, :a] + n_r new phones + orig_phone[r, b:]``, n_r = Tp_e - Tp_o + (b - a) >= 0.

        The kept phones are pinned to their original durations inside the ADM loop (1..127 each) and the new ones are
        decoded after them; ``span_frames`` (B,) gives the new phones exactly that many frames in all (``span_frames`` =
        L_o, the replaced phones' frames, keeps every later frame where it was), and ``duration_scale`` scales the new
        phones' predictions, both through ``synthesize``'s duration control.  The prosody LM then decodes only the
        8-frame blocks that overlap the new frames or straddle one of their ends; the other blocks keep the original's
        codes as pins of ``MegaPLM.infer`` (megatts2_b200/edit.py states the rule), and steps pinned in every row are not
        run.  ``sampling``, ``keys``, ``plm_context`` and ``check_range`` are ``synthesize``'s.

        Returns what ``synthesize`` returns: the whole edited utterance.  MRTE's latent depends on the whole phone
        sequence, and the mel decoder and vocoder see +-20 / +-14 frames around each frame, so samples outside the span
        move slightly; splicing into the original audio is the caller's choice.  ``return_intermediates`` adds
        ``edit_frames`` (B, 2), [F_a, F_a + L_n): the regenerated frames (sample 256 (5 + f) is frame f), and
        ``code_pins`` (B, T) the pins used.  Every argument is checked on the host before any device work; the
        arguments ``synthesize`` takes for what an edit sets itself, or does not support, are rejected by name."""
        for k in rejected:
            if k in ED.REJECTED:
                raise L.MttsError(f"edit does not take {k}: an edit sets the durations and codes around the span "
                                  "itself, on the reference-faithful decodes without a prosody mix or a prompt re-vocode, "
                                  "and keeps the original voice")
        if rejected:
            raise TypeError(f"edit() got unexpected keyword argument(s) {sorted(rejected)}")
        plan = ED.EditPlan(phone_tokens, orig_phone, orig_durations, orig_codes, span, span_frames, self.plm.vq_bins)
        dev = phone_tokens.device
        control = _duration_control(phone_tokens, None, False, duration_scale, plan.total_frames, plan.pinned_durations)
        args = (phone_tokens, mels, None, False, None, None, sampling, keys, None, None, None, plm_context, control,
                plan.code_pins)
        out = self._synthesize(*args)
        if check_range and _fp16_operands() and ops.tc_overflow(dev):
            _warn_fp16_range("re-running this batch on the bf16x3 engine")
            with pack.engine_scope(pack.ENGINE_BF16X3):
                out = self._synthesize(*args)
        if return_intermediates:
            out["edit_frames"] = plan.edit_frames(out["totals"])
            out["code_pins"] = plan.code_pins(out["totals"], out["p_codes"].shape[1])
            return out
        return (out["wav"], out["wav_lens"]) if return_lengths else out["wav"]

    def _revocode_cfg(self):
        """(V, frac, start) of the overlapped prompt re-vocode: V = SM budget of the side stream (MEGATTS2_REVOCODE_SMS; 0 = run
        the re-vocode after the synthesis on the calling stream), frac = share of the batch's prompts re-vocoded there
        (MEGATTS2_REVOCODE_FRAC; the rest follows sequentially at full width), start = 'mrte' | 'adm': the first stage of the
        calling stream that runs beside it, on the remaining SMs (MEGATTS2_REVOCODE_FROM)."""
        import os
        return (int(os.environ.get("MEGATTS2_REVOCODE_SMS", str(REVOCODE_SMS_DEFAULT))),
                float(os.environ.get("MEGATTS2_REVOCODE_FRAC", str(REVOCODE_FRAC_DEFAULT))),
                os.environ.get("MEGATTS2_REVOCODE_FROM", REVOCODE_FROM_DEFAULT))

    def _check_prosody(self, phone_tokens, prosody_mels, prosody_weights, causal_decode, duration_weights=None,
                       plm_context=None):
        if plm_context is not None and prosody_mels is not None:
            raise L.MttsError("plm_context does not combine with prosody_mels: the mixed sources would need one code "
                              "history with one context length")
        if prosody_mels is None:
            if prosody_weights is not None:
                raise L.MttsError("prosody_weights without prosody_mels")
            if duration_weights is not None:
                raise L.MttsError("duration_weights without prosody_mels")
            return
        if causal_decode:
            raise L.MttsError("prosody interpolation runs on the reference-faithful decode, not with causal_decode=True")
        if isinstance(prosody_mels, torch.Tensor) or not len(prosody_mels):
            raise L.MttsError("prosody_mels must be a non-empty list of (B, Tm, mel_bins) tensors")
        if prosody_weights is None:
            raise L.MttsError("prosody_mels needs prosody_weights: (K,) or (B, K), K = 1 + len(prosody_mels)")
        B, nb = phone_tokens.shape[0], self.generator.mrte.mel_bins
        for k, m in enumerate(prosody_mels):
            ops._dev(m, name=f"prosody_mels[{k}]")
            if m.dim() != 3 or m.shape[0] != B or m.shape[2] != nb or m.shape[1] < 1:
                raise L.MttsError(f"prosody_mels[{k}]: expected ({B}, Tm, {nb}), got {tuple(m.shape)}")
        S.synth_mix_weights(prosody_weights, 1 + len(prosody_mels), B, phone_tokens.shape[1], "prosody mix")
        if duration_weights is not None:
            S.synth_mix_weights(duration_weights, 1 + len(prosody_mels), B, phone_tokens.shape[1], "duration mix")

    def _check_timbre(self, phone_tokens, timbre_mels, timbre_weights):
        """-> (timbre_mels, their validated (B, K) or (B, Tp, K) CPU weights), or None without a timbre mix."""
        if timbre_mels is None and timbre_weights is None:
            return None
        if timbre_mels is None:
            raise L.MttsError("timbre_weights without timbre_mels")
        if isinstance(timbre_mels, torch.Tensor) or not len(timbre_mels):
            raise L.MttsError("timbre_mels must be a non-empty list of (B, Tm, mel_bins) tensors")
        if timbre_weights is None:
            raise L.MttsError("timbre_mels needs timbre_weights: (K,), (B, K) or (B, Tp, K), K = 1 + len(timbre_mels)")
        K = 1 + len(timbre_mels)
        if K > S.MIX_MAX_SOURCES:
            raise L.MttsError(f"timbre_mels: {K - 1} prompts, at most {S.MIX_MAX_SOURCES - 1} (K = 1 + len(timbre_mels) "
                              f"<= {S.MIX_MAX_SOURCES})")
        B, Tp = phone_tokens.shape
        check_prompts(timbre_mels, B, self.generator.mrte.mel_bins, "timbre_mels", phone_tokens.device)
        return list(timbre_mels), S.synth_mix_weights(timbre_weights, K, B, Tp, "timbre_weights")

    def _mrte(self, phone_tokens, mels, prosody_mels=None, timbre=None, mel_context=None):
        """The call's one MRTE pass -> (tc_latent of ``mels``, the latent of each prosody prompt or None, the timbre blend
        or None).  Without prompts it is ``mrte.tc_latent(phone_tokens, mels)``.  With them the phone encoder runs once
        (``MRTE.attend`` over [mels, *timbre_mels, the other prosody prompts]): a prosody prompt that is ``mels`` or one of
        ``timbre_mels`` (the same tensor object) is not encoded again.  Every latent is ``tc_latent(phone_tokens, its mel)``
        bit for bit, and the blend is ``MRTE.tc_latent_mix`` over [mels, *timbre_mels].  ``mel_context``:
        ``MRTE.encode_prompt(mels)``, computed once for several calls (a passage's sentences), so ``mels`` is not encoded
        here."""
        mrte = self.generator.mrte
        if prosody_mels is None and timbre is None:
            if mel_context is not None:
                return mrte.tc_latent(phone_tokens, mel_context=mel_context), None, None
            return mrte.tc_latent(phone_tokens, mels), None, None
        srcs = [mels] + (timbre[0] if timbre is not None else [])
        slot = {}
        for k, m in enumerate(srcs):
            slot.setdefault(id(m), k)
        for m in prosody_mels or ():
            if id(m) not in slot:
                slot[id(m)] = len(srcs)
                srcs.append(m)
        ys = mrte.attend(phone_tokens, srcs, None if mel_context is None else [mel_context] + [None] * (len(srcs) - 1))
        lat = {}

        def latent(k):
            if k not in lat:
                lat[k] = mrte.norm_relu(ys[k])
            return lat[k]
        prosody = None if prosody_mels is None else [latent(slot[id(m)]) for m in prosody_mels]
        blend = None if timbre is None else mrte.norm_relu_mix(ys[:1 + len(timbre[0])], timbre[1])
        return latent(0), prosody, blend

    def _synthesize(self, phone_tokens, mels, forced_durations, causal_decode, prompt_mels, overlap_prompt=None,
                    sampling=None, keys=None, prosody_mels=None, prosody_weights=None, duration_weights=None,
                    plm_context=None, control=None, code_pins=None, timbre=None, mel_context=None, mel_only=False):
        # ``code_pins`` (speech editing): totals, T -> the (B, T) code pins of MegaPLM.infer, built once the frame totals
        # are on the host.  ``mel_context`` (long-form synthesis): ``MRTE.encode_prompt(mels)``, encoded once per passage.
        # ``mel_only`` stops after the mel decoder: the result has no ``wav`` or ``wav_lens``.
        # The prompt re-vocode (:371-372) depends on nothing the synthesis computes, and the ADM loop (latency-bound: ~4 k short
        # dependent launches that fill a fraction of the SMs) leaves most of the device idle: the re-vocode is enqueued first,
        # on a side stream with an SM budget of V, and MRTE + ADM run beside it on the other SMs.  ops.launch_policy carries
        # the rules that make two streams share the device (csrc/conv_tc.cu, set_launch_policy): complementary budgets and
        # no programmatic dependent launch on the vocoder's stream.  The calling stream joins
        # the side stream before the first full-width stage (length regulator -> PLM), so nothing sized for the whole device is
        # ever enqueued while the vocoder's persistent CTAs hold SMs.
        pw_side, side, n_side = None, None, 0
        V, frac, start = self._revocode_cfg()
        dev = phone_tokens.device
        overlap = prompt_mels is not None and overlap_prompt is not False and (V > 0 or overlap_prompt is True)
        adm_decode = self.adm.infer_causal if causal_decode else self.adm.infer
        plm_decode = self.plm.infer_causal if causal_decode else self.plm.infer
        if overlap:
            nsm = ops.sm_count(dev)
            V = max(8, min(V if V > 0 else (2 * nsm) // 3, nsm - 8))
            n_side = max(1, min(prompt_mels.shape[0], int(round(prompt_mels.shape[0] * frac))))
            self.hifi_gan.generator._plan_get()          # weights are packed on the calling stream, before the fork
            main = torch.cuda.current_stream(dev)
            if getattr(self, "_side_stream", None) is None:
                self._side_stream = torch.cuda.Stream(device=dev)
            side = self._side_stream
            if start == "adm":
                tc_latent, lats, timbre_lat = self._mrte(phone_tokens, mels, prosody_mels, timbre, mel_context)
            side.wait_stream(main)
            prompt_mels.record_stream(side)
            with torch.cuda.stream(side), ops.launch_policy(V, pairs=True, pdl=False):
                pw_side = self.hifi_gan.decode_batch_cl(prompt_mels[:n_side])
            with ops.launch_policy(nsm - V, pairs=False, pdl=True):
                if start != "adm":
                    tc_latent, lats, timbre_lat = self._mrte(phone_tokens, mels, prosody_mels, timbre, mel_context)
                dt = self._durations(adm_decode, tc_latent, lats, duration_weights, control)
            main.wait_stream(side)
            pw_side.record_stream(main)
        else:
            tc_latent, lats, timbre_lat = self._mrte(phone_tokens, mels, prosody_mels, timbre, mel_context)
            dt = self._durations(adm_decode, tc_latent, lats, duration_weights, control)
        tc_expand, totals, src, step_w, dec_expand = self._plm_source(tc_latent, dt, forced_durations, phone_tokens, lats,
                                                                      prosody_weights, timbre_lat)
        if prosody_mels is not None:
            tc8 = src[0]
            p_codes = self.plm.infer_mix(src, prosody_weights if step_w is None else step_w, sampling=sampling, keys=keys)
        else:
            tc8 = src
            kw = {} if code_pins is None else {"pinned": code_pins(totals, tc8.shape[1])}
            p_codes = plm_decode(src, sampling=sampling, keys=keys, context=plm_context, **kw)
        B, Lmax = tc_expand.shape[0], tc_expand.shape[1]
        hop = HIFIGAN_HOP_LENGTH
        pad = self.hifi_gan.generator.cfg["inference_padding"]
        if mel_only:
            return dict(tc_latent=tc_latent, dt=dt, tc_latent_expand=tc_expand, tc8=tc8, p_codes=p_codes,
                        mel=self._decode_mel(dec_expand, p_codes, totals), totals=totals)
        if all(t == Lmax for t in totals):
            mel = self.generator.decode_mel_cl(dec_expand, p_codes)   # (B, L, 80) channels-last
            wav = self.hifi_gan.decode_batch_cl(mel)
        else:
            # ragged totals: decoder + vocoder per group of equal length (exactly the reference's batch-1 results)
            mel = torch.zeros(B, Lmax, self.generator.mrte.mel_bins, dtype=torch.float32, device=tc_expand.device)
            wav = torch.zeros(B, 1, hop * (Lmax + 2 * pad), dtype=torch.float32, device=tc_expand.device)
            for Lg in sorted(set(totals)):
                idx = torch.tensor([i for i, t in enumerate(totals) if t == Lg], device=tc_expand.device)
                if Lg == 0:
                    continue
                mg = self.generator.decode_mel_cl(dec_expand[idx, :Lg].contiguous(), p_codes[idx, :(Lg + 7) // 8].contiguous())
                wg = self.hifi_gan.decode_batch_cl(mg)
                mel[idx, :Lg] = mg
                wav[idx, :, :wg.shape[-1]] = wg
        wav_lens = [hop * (t + 2 * pad) for t in totals]
        if prompt_mels is not None:
            if pw_side is None:
                pw = self.hifi_gan.decode_batch_cl(prompt_mels)       # (B, 1, hop*(Tq + 2 pad))   (:371-372)
            elif n_side < prompt_mels.shape[0]:
                pw = torch.cat([pw_side, self.hifi_gan.decode_batch_cl(prompt_mels[n_side:])], dim=0)
            else:
                pw = pw_side
            wav = torch.cat([pw, wav], dim=-1)                        # (:373)
            wav_lens = [n + pw.shape[-1] for n in wav_lens]
        out = dict(tc_latent=tc_latent, dt=dt, tc_latent_expand=tc_expand, tc8=tc8, p_codes=p_codes,
                   mel=mel, wav=wav, totals=totals, wav_lens=wav_lens)
        if step_w is not None:
            out["prosody_step_weights"] = step_w
        if timbre_lat is not None:
            out["timbre_latent"] = timbre_lat
        return out

    def _decode_mel(self, dec_expand, p_codes, totals):
        """The mel decoder of ``_synthesize`` without the vocoder: one launch sequence when every total is Lmax, else one
        per group of equal totals (zero rows past a total)."""
        B, Lmax = dec_expand.shape[0], dec_expand.shape[1]
        if all(t == Lmax for t in totals):
            return self.generator.decode_mel_cl(dec_expand, p_codes)
        mel = torch.zeros(B, Lmax, self.generator.mrte.mel_bins, dtype=torch.float32, device=dec_expand.device)
        for Lg in sorted(set(totals) - {0}):
            idx = torch.tensor([i for i, t in enumerate(totals) if t == Lg], device=dec_expand.device)
            mel[idx, :Lg] = self.generator.decode_mel_cl(dec_expand[idx, :Lg].contiguous(),
                                                         p_codes[idx, :(Lg + 7) // 8].contiguous())
        return mel

    def _durations(self, adm_decode, tc_latent, prosody_latents, duration_weights, control=None):
        """-> dt (B, Tp) int32.  Without ``duration_weights``: ``adm_decode`` on ``tc_latent``.  With them:
        ``MegaADM.infer_mix`` over [tc_latent, *prosody_latents] (the prosody prompts' latents of ``_mrte``).  ``control``, the validated
        (scale, total, pins) of ``_duration_control``: the pins go into the ADM loop, and with a scale or a total the
        durations are ``ops.fit_durations`` of the decode's raw values."""
        scale, total, pins = control if control is not None else (None, None, None)
        fit = scale is not None or total is not None
        kw = {} if pins is None else {"pinned": pins}
        if fit:
            kw["return_raw"] = True
        if duration_weights is None:
            out = adm_decode(tc_latent, **kw)
        else:
            out = self.adm.infer_mix([tc_latent] + prosody_latents, duration_weights, **kw)
        if fit:
            return ops.fit_durations(out[1], scale, total, pins)
        return out[..., 0]

    def _plm_source(self, tc_latent, dt, forced_durations, phone_tokens, prosody_latents=None, prosody_weights=None,
                    timbre_latent=None):
        """The synthesis front end between the ADM and the PLM: the durations (``forced_durations`` if given, else
        ``dt``) expand ``tc_latent`` to frames -> (tc_expand (B, Lmax, tc_dim), the per-utterance frame totals on the host
        (one host sync), the PLM's source, the PLM's step weights, the mel decoder's latent frames).  The source is tc8,
        tc_expand max-pooled by 8, or with ``prosody_latents`` (the prosody prompts' latents of ``_mrte``) the list
        [tc8, *each latent length-regulated with the same durations to Lmax frames and max-pooled by 8].  The step weights
        are None unless ``prosody_weights`` has one row per phone; then they are its (B, ceil(Lmax / 8), K) expansion by
        the same durations (``ops.mix_step_weights``).  The decoder's frames are tc_expand, or ``timbre_latent``
        length-regulated with the same durations to Lmax frames."""
        d_used = dt if forced_durations is None else forced_durations.to(dt.device, torch.int32)
        tc_expand, totals = ops.length_regulate(tc_latent, d_used, return_host_totals=True)   # one host sync
        tc8 = ops.maxpool_time(tc_expand, 8)
        Lmax = tc_expand.shape[1]
        dec_expand = tc_expand if timbre_latent is None else ops.length_regulate(timbre_latent, d_used, l_out=Lmax)[0]
        if prosody_latents is None:
            return tc_expand, totals, tc8, None, dec_expand
        src = [tc8] + [ops.maxpool_time(ops.length_regulate(lat, d_used, l_out=Lmax)[0], 8) for lat in prosody_latents]
        step_w = None
        if S.per_step(prosody_weights):
            B, Tp = phone_tokens.shape
            pw = S.mix_step_weights(prosody_weights, len(src), B, Tp).to(tc8.device)
            step_w = ops.mix_step_weights(pw, d_used, tc8.shape[1])
        return tc_expand, totals, src, step_w, dec_expand

    def synthesize_stream(self, phone_tokens: torch.Tensor, mels: torch.Tensor, forced_durations: torch.Tensor = None,
                          prompt_mels: torch.Tensor = None, sampling: S.Sampling = None, keys=None, check_range: bool = True,
                          chunk_frames: int = 64, prosody_mels=None, prosody_weights=None, duration_weights=None,
                          plm_context=None, duration_scale=None, total_frames=None, pinned_durations=None,
                          timbre_mels=None, timbre_weights=None, **unsupported):
        """``synthesize`` as a generator of waveform chunks, each yielded as soon as the prosody LM has decoded the codes
        its samples depend on.  Arguments as in ``synthesize``; ``chunk_frames`` mel frames (hop = 256 samples each) per
        chunk.  Each chunk is a dict: ``wav`` (B, 1, n) device tensor, ``offset`` (its first sample's index in the waveform
        ``synthesize`` returns), ``valid`` (per utterance, the samples of this chunk inside its waveform; the rest are
        zeros), ``last``; the last chunk also has ``p_codes``, ``dt``, ``mel`` and ``wav_lens``.  With ``prompt_mels`` the
        first chunk is the re-vocoded prompt.  The chunks, concatenated, are ``synthesize``'s waveform (same codes and
        durations; samples within rounding: a window can take another tensor-core plan than the whole sequence).

        The stream runs MRTE and the ADM, then alternates a PLM range (``MegaPLM.decode_until``), the mel rows that range
        made computable (decoder windows with a halo of ``generator.decoder.receptive_field()`` frames) and the chunk's
        vocoder window (halo ``hifi_gan.generator.receptive_field()``); megatts2_b200/stream.py has the schedule.  Ragged
        totals: the utterances whose clipped windows are equal run as one batch.

        ``check_range`` (fp16 operand engines): the range flag is read after every PLM range and every chunk, and nothing
        is yielded before the first read.  Raised before the first synthesized chunk is yielded: the stream warns and
        restarts on bf16x3, and then equals ``synthesize``'s rerun.  Raised later: it warns, recomputes the current step on
        bf16x3 and finishes there, keeping the codes and chunks it has emitted - so such a stream can differ from
        ``synthesize``, which reruns the whole batch.  ``causal_decode`` and ``overlap_prompt`` are not supported."""
        if unsupported:
            raise L.MttsError(f"synthesize_stream: unsupported argument(s) {sorted(unsupported)} "
                              "(the causal decode and the overlapped prompt re-vocode are not streamed)")
        if int(chunk_frames) < 1:
            raise L.MttsError(f"synthesize_stream: chunk_frames must be >= 1, got {chunk_frames}")
        self._check_prosody(phone_tokens, prosody_mels, prosody_weights, False, duration_weights, plm_context)
        control = _duration_control(phone_tokens, forced_durations, False, duration_scale, total_frames,
                                    pinned_durations)
        timbre = self._check_timbre(phone_tokens, timbre_mels, timbre_weights)
        guard = check_range and _fp16_operands()
        return self._stream_outer(phone_tokens, mels, forced_durations, prompt_mels, sampling, keys, guard,
                                  int(chunk_frames), (prosody_mels, prosody_weights, duration_weights, plm_context),
                                  control, timbre)

    def _stream_outer(self, phone_tokens, mels, forced_durations, prompt_mels, sampling, keys, guard, chunk_frames,
                      prosody, control, timbre):
        try:
            yield from self._stream(phone_tokens, mels, forced_durations, prompt_mels, sampling, keys, guard, chunk_frames,
                                    prosody, control, timbre)
        except _RangeRestart:
            _warn_fp16_range("restarting this stream on the bf16x3 engine")
            yield from self._stream(phone_tokens, mels, forced_durations, prompt_mels, sampling, keys, False, chunk_frames,
                                    prosody, control, timbre, engine=pack.ENGINE_BF16X3)

    def _stream(self, phone_tokens, mels, forced_durations, prompt_mels, sampling, keys, guard, chunk_frames, prosody,
                control, timbre, engine=None):
        # The engine scope is entered around each computing step only, never across a yield: the caller's own work between
        # chunks keeps its engine.
        from .. import stream as SCH
        import contextlib

        def scope():
            return pack.engine_scope(engine) if engine is not None else contextlib.nullcontext()

        dev = phone_tokens.device
        gen, voc = self.generator, self.hifi_gan.generator
        hop, pad = HIFIGAN_HOP_LENGTH, voc.cfg["inference_padding"]
        hd, hv = gen.decoder.receptive_field(), voc.receptive_field()
        with torch.no_grad(), scope():
            prosody_mels, prosody_weights, duration_weights, plm_context = prosody
            tc_latent, lats, timbre_lat = self._mrte(phone_tokens, mels, prosody_mels, timbre)
            dt = self._durations(self.adm.infer, tc_latent, lats, duration_weights, control)
            tc_expand, totals, src, step_w, dec_expand = self._plm_source(tc_latent, dt, forced_durations, phone_tokens,
                                                                          lats, prosody_weights, timbre_lat)
            dec = self.plm.begin_decode(src, sampling=sampling, keys=keys,
                                        weights=prosody_weights if step_w is None else step_w, context=plm_context)
            pw = self.hifi_gan.decode_batch_cl(prompt_mels) if prompt_mels is not None else None
        B, Lmax, T = tc_expand.shape[0], tc_expand.shape[1], dec.T
        if Lmax < 1:
            raise L.MttsError("synthesize_stream: every utterance has zero frames")
        mel = torch.zeros(B, Lmax, gen.mrte.mel_bins, dtype=torch.float32, device=dev)
        plans = [SCH.schedule(t, chunk_frames, hd, hv, pad, Lmax) for t in totals]
        P = SCH.chunk_positions(Lmax, chunk_frames, pad)
        K = len(P) - 1
        off0 = 0 if pw is None else pw.shape[-1]
        emitted = False

        def flag_raised():
            nonlocal guard, engine
            if not guard or not ops.tc_overflow(dev):
                return False
            if not emitted:
                raise _RangeRestart()
            _warn_fp16_range("finishing this stream on the bf16x3 engine (its chunks can differ from synthesize's rerun)")
            guard, engine = False, pack.ENGINE_BF16X3
            return True

        def groups(k, key):
            """utterances with equal key(chunk) for chunk k -> [(key, index tensor or slice)]"""
            by = {}
            for i, pl in enumerate(plans):
                c = pl[k]
                if c is not None and key(c) is not None:
                    by.setdefault(key(c), []).append(i)
            return [(kk, slice(None) if len(ids) == B else torch.tensor(ids, device=dev)) for kk, ids in by.items()]

        def synth_chunk(k):
            n = hop * (P[k + 1] - P[k])
            wav = torch.zeros(B, 1, n, dtype=torch.float32, device=dev)
            for (rows, win), idx in groups(k, lambda c: (c.rows, c.dec) if c.dec is not None else None):
                (r0, r1), (da, db) = rows, win
                m = gen.decode_mel_cl(dec_expand[idx, da:db].contiguous(), dec.target[idx, da // 8:-(-db // 8)])
                mel[idx, r0:r1] = m[:, r0 - da:r1 - da]
            for (p0, p1, va, vb), idx in groups(k, lambda c: (c.p0, c.p1) + c.voc):
                w = self.hifi_gan.decode_batch_cl(mel[idx, va:vb])
                wav[idx, :, :hop * (p1 - p0)] = w[:, :, hop * (p0 - va):hop * (p1 - va)]
            return wav

        for k in range(K):
            t_need = T if k == K - 1 else max(pl[k].t1 for pl in plans if pl[k] is not None)
            while True:
                t_prev = dec.t
                with torch.no_grad(), scope():
                    self.plm.decode_until(dec, max(t_need, dec.t))
                if not flag_raised():
                    break
                dec.t = t_prev                               # redo this range on bf16x3
            while True:
                with torch.no_grad(), scope():
                    wav = synth_chunk(k)
                if not flag_raised():
                    break
            if pw is not None and not emitted:
                yield dict(wav=pw, offset=0, valid=[pw.shape[-1]] * B, last=False)
            emitted = True
            valid = [0 if pl[k] is None else hop * (pl[k].p1 - pl[k].p0) for pl in plans]
            chunk = dict(wav=wav, offset=off0 + hop * P[k], valid=valid, last=k == K - 1)
            if k == K - 1:
                chunk.update(p_codes=dec.target.clone(), dt=dt, mel=mel,
                             wav_lens=[hop * (t + 2 * pad) + off0 for t in totals])
            yield chunk

    @torch.no_grad()
    def synthesize_passage(self, sentences, mels, pause_frames=0, context_rows: int = 128, plm_context=None,
                           forced_durations=None, duration_scale=None, sampling: S.Sampling = None, keys=None,
                           check_range: bool = True, return_lengths: bool = False, return_intermediates: bool = False,
                           **rejected):
        """Long-form synthesis: a passage of S sentences, each decoded with the sentences before it as the prosody LM's
        context, vocoded as one waveform.  ``sentences``: S phone tensors (B, Tp_i) int64 on one device; row b of each
        belongs to passage b (B voices or takes of one text).  ``mels`` (B, Tm, 80): the voice prompt, encoded once.

        Sentence i runs what ``synthesize(sentences[i], mels, plm_context=W_i)`` runs up to the mel decoder: MRTE and
        the ADM see the sentence alone, the regime they were trained on.  W_i is the last P_i = min(context_rows, min_b
        H_b) rows of each row's history: the rows of ``plm_context`` (Bc = 1 or B), then each earlier sentence's
        ceil(L / 8) valid max-pooled latents and codes (megatts2_b200/passage.py states the rule).  The window is
        bounded, so the cost is linear in S.  The default of 128 rows (1024 mel frames, about 16 s at 16 kHz: several
        sentences) costs about 1.1x the plain PLM decode at B = 1 and 4.4x at B = 64 (DESIGN.md section 7);
        ``context_rows=0`` makes the sentences independent.  Sampled sentence i of row b draws with the key
        ``keys[b] + i * 2^32``, so sentence 0 is ``synthesize``'s take and no two sentences share noise.

        Row b's passage mel is its sentences' frames with ``pause_frames`` (an int, or (B, S - 1) ints >= 0) frames of
        silence (log 1e-5, the front end's floor) after each but the last; the vocoder runs once over it, per group of
        equal passage length, so sentence edges are ordinary frames to it.  ``forced_durations``: None or one (B, Tp_i)
        tensor per sentence; ``duration_scale``: a number or (B,); they do not combine.  ``check_range``: the range flag
        is read after the prompt's encoding, each sentence and the vocoder, and a raised flag redoes that piece alone on
        bf16x3.  The AR decodes run eagerly: the callers' CUDA-graph caches are left as they were.

        -> wav (B, 1, 256 (max F + 10)) [, wav_lens with ``return_lengths``: 256 (F_b + 10)]; ``return_intermediates``
        gives a dict with ``wav``, ``wav_lens``, ``mel`` (B, max F, 80), ``frame_offsets`` (B, S) (sentence i of row b
        starts at frame f, sample 256 (5 + f)), ``context_rows_used`` (S,) and ``sentences`` (per sentence ``dt``,
        ``p_codes``, ``tc8``, ``totals``).  Every argument is checked on the host before any device work;
        ``synthesize``'s arguments a passage does not take are rejected by name."""
        plan = self._passage_plan(sentences, mels, pause_frames, context_rows, plm_context, forced_durations,
                                  duration_scale, sampling, keys, rejected)
        guard = check_range and _fp16_operands()
        B, hop, pad = plan.B, HIFIGAN_HOP_LENGTH, self.hifi_gan.generator.cfg["inference_padding"]
        pm = PS.PassageMel(B, self.generator.mrte.mel_bins, plan.device)
        sents, used = [], []
        for i, (out, P) in enumerate(PS.run_sentences(self, plan, guard)):
            pm.place(out["mel"], out["totals"], [p[i] for p in plan.pauses] if i < plan.S - 1 else None)
            sents.append({k: out[k] for k in ("dt", "p_codes", "tc8", "totals")})
            used.append(P)
        offsets, F = PS.frame_offsets([s["totals"] for s in sents], plan.pauses)
        Fmax = max(F)
        mel = pm.buf[:, :Fmax]
        wav = torch.zeros(B, 1, hop * (Fmax + 2 * pad), dtype=torch.float32, device=plan.device)
        live = [b for b in range(B) if F[b] > 0]
        for n, (ids, w) in PS.vocode(self, mel, live, [F[b] for b in live], guard).items():
            if len(ids) == B:
                wav = w
            else:
                wav[torch.tensor(ids, device=plan.device), :, :w.shape[-1]] = w
        wav_lens = [hop * (f + 2 * pad) for f in F]
        if return_intermediates:
            return dict(wav=wav, wav_lens=wav_lens, mel=mel, frame_offsets=torch.tensor(offsets, dtype=torch.int64),
                        context_rows_used=torch.tensor(used, dtype=torch.int64), sentences=sents)
        return (wav, wav_lens) if return_lengths else wav

    def synthesize_passage_stream(self, sentences, mels, pause_frames=0, context_rows: int = 128, plm_context=None,
                                  forced_durations=None, duration_scale=None, sampling: S.Sampling = None, keys=None,
                                  check_range: bool = True, **rejected):
        """``synthesize_passage`` as a generator of chunks, one per sentence; every argument is checked before the first
        ``next``.  Chunk i holds each row's samples of the pause before sentence i and of sentence i (the first chunk
        also the vocoder's leading padding, the last its trailing padding), from a vocoder window with a halo of
        ``hifi_gan.generator.receptive_field()`` frames on each side.  It is yielded as soon as the passage mel covers
        its window in every row: right after sentence i when the pause after it is at least the halo in every row,
        else after sentence i + 1.  Each chunk is a dict: ``wav`` (B, 1, n), ``offset`` and ``valid`` (per row: where
        its samples start in ``synthesize_passage``'s waveform, and how many of the chunk's first samples are that
        row's; the rest are zeros), ``sentence`` (i) and ``last``; the last chunk also has ``wav_lens``, ``mel`` and
        ``frame_offsets``.  Rows whose windows are equal share one vocoder batch.  Put together, the chunks are
        ``synthesize_passage``'s waveform within rounding (a window can take another tensor-core plan than the whole
        passage); codes, durations and mel are the same bit for bit.  ``check_range`` redoes a sentence or a chunk's
        vocoder launches on bf16x3, as ``synthesize_passage`` does."""
        plan = self._passage_plan(sentences, mels, pause_frames, context_rows, plm_context, forced_durations,
                                  duration_scale, sampling, keys, rejected)
        return self._passage_stream(plan, check_range and _fp16_operands())

    def _passage_plan(self, sentences, mels, pause_frames, context_rows, plm_context, forced_durations, duration_scale,
                      sampling, keys, rejected):
        return PS.PassagePlan(sentences, mels, pause_frames, context_rows, plm_context, forced_durations,
                              duration_scale, sampling, keys, self.plm.vq_bins, self.plm.tc_latent_dim,
                              self.generator.mrte.mel_bins, rejected)

    def _passage_stream(self, plan, guard):
        import contextlib
        B, S_, dev = plan.B, plan.S, plan.device
        hop, pad = HIFIGAN_HOP_LENGTH, self.hifi_gan.generator.cfg["inference_padding"]
        hv = self.hifi_gan.generator.receptive_field()
        pm = PS.PassageMel(B, self.generator.mrte.mel_bins, dev)
        totals, nxt = [], 0

        def chunk(i, final):
            """chunk i, or None while its window is not covered in every row"""
            offsets, F = PS.frame_offsets(totals + [[0] * B] * (S_ - len(totals)), plan.pauses)
            bounds = PS.chunk_bounds(offsets, totals + [[0] * B] * (S_ - len(totals)), F, i, pad)
            wins = [PS.vocoder_window(p0, p1, pad, hv, pm.f[b], final) for b, (p0, p1) in enumerate(bounds)]
            if any(w is None for b, w in enumerate(wins) if bounds[b][1] > bounds[b][0]):
                return None
            valid = [hop * max(p1 - p0, 0) for p0, p1 in bounds]
            wav = torch.zeros(B, 1, max(valid), dtype=torch.float32, device=dev)
            groups = {}
            for b, ((p0, p1), w) in enumerate(zip(bounds, wins)):
                if p1 > p0 and w[1] > w[0]:
                    groups.setdefault((p0, p1) + w, []).append(b)
            redo = False
            while True:
                with pack.engine_scope(pack.ENGINE_BF16X3) if redo else contextlib.nullcontext():
                    for (p0, p1, va, vb), ids in groups.items():
                        idx = slice(None) if len(ids) == B else torch.tensor(ids, device=dev)
                        w = self.hifi_gan.decode_batch_cl(pm.buf[idx, va:vb])
                        wav[idx, :, :hop * (p1 - p0)] = w[:, :, hop * (p0 - va):hop * (p1 - va)]
                if redo or not (guard and ops.tc_overflow(dev)):
                    break
                _warn_fp16_range(f"re-running the vocoder of chunk {i} of this passage on the bf16x3 engine")
                redo = True
            out = dict(wav=wav, offset=[hop * p0 for p0, _ in bounds], valid=valid, sentence=i, last=i == S_ - 1)
            if i == S_ - 1:
                out.update(wav_lens=[hop * (f + 2 * pad) for f in F], mel=pm.buf[:, :max(F)],
                           frame_offsets=torch.tensor(offsets, dtype=torch.int64))
            return out

        for i, (out, _) in enumerate(PS.run_sentences(self, plan, guard)):
            with torch.no_grad():
                pm.place(out["mel"], out["totals"], [p[i] for p in plan.pauses] if i < S_ - 1 else None)
            totals.append(out["totals"])
            while nxt <= i:
                with torch.no_grad():
                    c = chunk(nxt, i == S_ - 1)
                if c is None:
                    break
                yield c
                nxt += 1

    @torch.no_grad()
    def synthesize_many(self, items, max_batch: int = 64, sampling: S.Sampling = None, **kw):
        """Ragged front door: ``items`` = list of (phone (Tp_i,) int64, prompt mel (Tm_i, 80)).  Utterances are
        bucketed by (Tp, Tm) - the MRTE phone encoder and the prompt encoder are unmasked in the reference
        (modules/mrte.py:154-171), so padding either would change results - and each bucket runs as one batch.
        Returns a list of 1-D waveforms (valid samples only), in input order.  With ``sampling``, utterance i is keyed
        by its index i in ``items``, so the bucketing and ``max_batch`` do not change what it draws.  Prosody prompts
        (``prosody_mels``) are not taken here: call ``synthesize`` per batch.  Of the duration controls only a scalar
        ``duration_scale`` is: the buckets regroup the utterances, so per-utterance values would not line up."""
        if "prosody_mels" in kw or "prosody_weights" in kw or "plm_context" in kw:
            raise L.MttsError("synthesize_many does not take prosody prompts or a PLM context; call synthesize per batch")
        if "timbre_mels" in kw or "timbre_weights" in kw:
            raise L.MttsError("synthesize_many does not take timbre_mels or timbre_weights (timbre prompts); call "
                              "synthesize per batch")
        if "total_frames" in kw or "pinned_durations" in kw:
            raise L.MttsError("synthesize_many does not take total_frames or pinned_durations (per-utterance values); "
                              "call synthesize per batch")
        if kw.get("duration_scale") is not None:
            kw["duration_scale"] = S.duration_scale(kw["duration_scale"], 1, 1)
            if kw["duration_scale"].dim() != 0:
                raise L.MttsError("synthesize_many takes a scalar duration_scale only")
        if sampling is not None:
            kw["sampling"] = sampling
        buckets = {}
        for i, (ph, m) in enumerate(items):
            buckets.setdefault((ph.shape[0], m.shape[0]), []).append(i)
        out = [None] * len(items)
        for _, ids in sorted(buckets.items()):
            for s in range(0, len(ids), max_batch):
                chunk = ids[s:s + max_batch]
                ph = torch.stack([items[i][0] for i in chunk])
                mm = torch.stack([items[i][1] for i in chunk])
                if sampling is not None:
                    kw["keys"] = torch.tensor(chunk, dtype=torch.int64)
                wav, lens = self.synthesize(ph, mm, return_lengths=True, **kw)
                for j, i in enumerate(chunk):
                    out[i] = wav[j, 0, :lens[j]]
        return out

    def forward(self, wavs_dir: str, text: str, out_path: str = 'test.wav'):
        """Reference signature (models/megatts2.py:325-375): prompt wavs + text -> writes test.wav.  The audio side
        (decode, resample to 16 kHz, peak normalisation, mel, wav writing) runs through megatts2_b200.audio on the device
        (SURVEY.md 8f-3); the text side needs the reference's host-side G2P (TextTokenizer / TokensCollector - out of the
        hot path) to be importable."""
        from .. import audio
        try:
            from modules.tokenizer import TextTokenizer          # the reference's host-side G2P
            from modules.datamodule import TokensCollector
        except Exception as e:   # pragma: no cover - host text front end is outside the hot path
            raise L.MttsError("Megatts.forward needs the reference's host-side text front end (G2P, TokensCollector): "
                              f"{e}; use synthesize() with phone tensors") from e
        dev = next(self.parameters()).device
        clips = [audio.read_wav(w) for w in glob.glob(f'{wavs_dir}/*.wav')]
        mels, mels_prompt = self.prompt_mels(clips)
        tt, ttc = TextTokenizer(), TokensCollector(self.symbol_table)
        phone_tokens = ttc.phone2token(tt.tokenize_lty(tt.tokenize(text))).unsqueeze(0).to(dev)
        audio_out = self.synthesize(phone_tokens, mels, prompt_mels=mels_prompt)
        audio.save_wav(out_path, audio_out[0], HIFIGAN_SR)

    def prompt_mels(self, clips):
        """The prompt loop of forward() (:333-346) for decoded clips [(float32 samples, sr)]: resample + normalise (one
        launch per sampling rate), mel per clip, concatenated along time -> (mels (1, sum frames, 80), first clip's mel
        (1, frames, 80))."""
        from .. import audio
        dev = next(self.parameters()).device
        wav, lens = audio.load_prompts(clips, dev, HIFIGAN_SR)
        per_clip = [extract_mel_spec(wav[i:i + 1, :n], frames_major=True)[0] for i, n in enumerate(lens.tolist())]
        return torch.cat(per_clip, 0).unsqueeze(0), per_clip[0].unsqueeze(0)
