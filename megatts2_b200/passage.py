"""Long-form synthesis's host side (``Megatts.synthesize_passage`` / ``synthesize_passage_stream``): the validated
passage, the prosody LM's context window, the sampling keys of each sentence, the layout of the passage mel and the
stream's chunks.

A passage is S sentences of B rows; row b of every sentence belongs to passage b.  Sentence i runs what
``synthesize(sentences[i], mels, plm_context=W_i)`` runs, up to the mel decoder.  The history of row b before sentence i
is the rows of the initial ``plm_context`` (if any), then, for each earlier sentence s, its ceil(L_{b,s} / 8) valid
max-pooled latent rows and their codes (L_{b,s}: that sentence's frame total in row b).  With H_b history rows,
W_i is the last P_i = min(context_rows, min_b H_b) rows of each row's history (no context when P_i = 0).  Only the last
``context_rows`` rows of a history are ever read, so a row keeps no more than that many: the cost of a sentence does
not grow with its position in the passage.

Row b's passage mel is sentence 0's L_{b,0} frames, ``pause[b][0]`` silence frames, sentence 1's frames, and so on.
Sentence i starts at frame f_{b,i}; the passage has F_b frames and its waveform 256 (F_b + 10) samples, sample
256 (5 + f) being frame f.

Stream chunk i of row b holds the pause before sentence i (none for i = 0) and sentence i's samples; the first chunk
also holds the vocoder's leading padding and the last its trailing padding.  A chunk therefore ends where its sentence
ends, and its vocoder window reaches ``hv`` frames (the vocoder's receptive field) past that: into the pause after it,
so the chunk is ready right after its sentence when that pause is at least ``hv`` frames in every row, and otherwise
once the next sentence's mel is placed.  (A chunk that also held the pause after its sentence would always wait for the
next sentence.)"""
import numpy as np
import torch

from . import _lib as L
from . import sampling as S

FRAMES_PER_CODE = 8
KEY_STRIDE = 1 << 32          # sentence i of row b draws with the key keys[b] + i * 2^32 (int64, wrapping)
SILENCE = float(np.log(np.float32(1e-5)))   # log(1e-5) in fp32: the mel front end's log floor, the mel of silence

# arguments of ``synthesize`` that a passage does not take, with the reason
REJECTED = {
    "prosody_mels": "prosody mixes inside a passage are not built (each sentence's prosody continues the passage)",
    "prosody_weights": "prosody mixes inside a passage are not built (each sentence's prosody continues the passage)",
    "duration_weights": "duration mixes inside a passage are not built",
    "timbre_mels": "timbre mixes inside a passage are not built; the passage keeps the voice of mels",
    "timbre_weights": "timbre mixes inside a passage are not built; the passage keeps the voice of mels",
    "total_frames": "a passage has no per-sentence target length; use forced_durations or duration_scale",
    "pinned_durations": "a passage has no per-sentence duration pins; use forced_durations",
    "causal_decode": "a passage runs the reference-faithful decodes, not the causal KV-cache decode",
    "prompt_mels": "a passage does not re-vocode and prepend a prompt; concatenate it yourself",
    "overlap_prompt": "a passage does not re-vocode and prepend a prompt",
}


def _wrap64(v):
    return (v + (1 << 63)) % (1 << 64) - (1 << 63)


def sentence_keys(keys, i):
    """The row keys of sentence i: keys[b] + i * 2^32 in wrapping int64 arithmetic (a list of B ints)."""
    return [_wrap64(k + i * KEY_STRIDE) for k in keys]


def window_rows(history, context_rows):
    """P = min(context_rows, min_b H_b): the context rows sentence i reads from each row's history of H_b rows."""
    return min([context_rows] + list(history)) if history else 0


def codes_rows(totals):
    """ceil(L / 8) per row: the valid max-pooled rows (and codes) of a sentence whose rows have L frames."""
    return [-(-int(t) // FRAMES_PER_CODE) for t in totals]


def history_update(kept, n, context_rows):
    """A row keeps the last min(context_rows, kept + n) rows of [its kept rows; the n new ones] -> (keep, o, m): it
    keeps o old rows (the last o of ``kept``) followed by the last m new rows."""
    keep = [min(context_rows, k + nb) for k, nb in zip(kept, n)]
    m = [min(nb, kp) for nb, kp in zip(n, keep)]
    return keep, [kp - mb for kp, mb in zip(keep, m)], m


def frame_offsets(totals, pauses):
    """totals[i][b] = L_{b,i} and pauses[b][i] (S - 1 per row) -> (offsets [b][i] = f_{b,i}, F [b] passage frames)."""
    S_, B = len(totals), len(totals[0]) if totals else 0
    offs, F = [], []
    for b in range(B):
        f, row = 0, []
        for i in range(S_):
            row.append(f)
            f += int(totals[i][b]) + (int(pauses[b][i]) if i < S_ - 1 else 0)
        offs.append(row)
        F.append(f)
    return offs, F


def chunk_bounds(offsets, totals, F, i, pad):
    """Positions [p0, p1) of stream chunk i in each row (position p: sample 256 p of the padded waveform; frame f owns
    position f + pad): from the end of sentence i - 1 (0 for the first chunk) to the end of sentence i (F + 2 pad for the
    last chunk)."""
    S_ = len(totals)
    out = []
    for b in range(len(F)):
        p0 = 0 if i == 0 else offsets[b][i - 1] + int(totals[i - 1][b]) + pad
        p1 = F[b] + 2 * pad if i == S_ - 1 else offsets[b][i] + int(totals[i][b]) + pad
        out.append((p0, p1))
    return out


def vocoder_window(p0, p1, pad, hv, F_known, final):
    """The mel frames [va, vb) a chunk at positions [p0, p1) is vocoded from, given F_known frames of the row placed so
    far (``final``: the row's whole passage is placed) -> (va, vb), or None while the window is not covered yet."""
    va = max(p0 - pad - hv, 0)
    va -= va % 8
    vb = p1 - pad + hv
    if vb > F_known:
        if not final:
            return None
        vb = F_known
    return min(va, max(vb - 1, 0)), vb


class PassagePlan:
    """A validated passage (every check on the host, before any device work).  Each error names the sentence and, where
    there is one, the row."""

    def __init__(self, sentences, mels, pause_frames, context_rows, plm_context, forced_durations, duration_scale,
                 sampling, keys, vq_bins, tc_dim, mel_bins, rejected):
        for k in rejected:
            if k in REJECTED:
                raise L.MttsError(f"synthesize_passage does not take {k}: {REJECTED[k]}")
        if rejected:
            raise TypeError(f"synthesize_passage() got unexpected keyword argument(s) {sorted(rejected)}")
        if isinstance(sentences, torch.Tensor) or not isinstance(sentences, (list, tuple)) or not sentences:
            raise L.MttsError("sentences must be a non-empty list of (B, Tp_i) int64 phone tensors")
        self.S = len(sentences)
        for i, ph in enumerate(sentences):
            if not isinstance(ph, torch.Tensor) or ph.dtype != torch.int64 or ph.dim() != 2 or ph.shape[1] < 1:
                raise L.MttsError(f"sentences[{i}]: expected a (B, Tp >= 1) int64 tensor, got "
                                  f"{getattr(ph, 'dtype', type(ph).__name__)} {tuple(getattr(ph, 'shape', ()))}")
            if ph.shape[0] != sentences[0].shape[0] or ph.device != sentences[0].device:
                raise L.MttsError(f"sentences[{i}]: {tuple(ph.shape)} on {ph.device}, expected B = "
                                  f"{sentences[0].shape[0]} rows on {sentences[0].device} like sentences[0]")
        self.B, self.device = sentences[0].shape[0], sentences[0].device
        B = self.B
        if self.B < 1:
            raise L.MttsError("sentences: B must be >= 1")
        if not (isinstance(mels, torch.Tensor) and mels.dtype == torch.float32 and mels.dim() == 3
                and mels.shape[0] == B and mels.shape[1] >= 1 and mels.shape[2] == mel_bins):
            raise L.MttsError(f"mels: expected a ({B}, Tm >= 1, {mel_bins}) float32 tensor, got "
                              f"{getattr(mels, 'dtype', type(mels).__name__)} {tuple(getattr(mels, 'shape', ()))}")
        if mels.device != self.device:
            raise L.MttsError(f"mels: on {mels.device}, expected {self.device} (the sentences' device)")
        if isinstance(context_rows, bool) or not isinstance(context_rows, (int, np.integer)) or context_rows < 0:
            raise L.MttsError(f"context_rows must be an int >= 0, got {context_rows!r}")
        self.context_rows = int(context_rows)
        self.pauses = self._pauses(pause_frames)
        self.context = self._context(plm_context, vq_bins, tc_dim)
        if forced_durations is not None and duration_scale is not None:
            raise L.MttsError("forced_durations replace the ADM's durations; they do not combine with duration_scale")
        self.forced = None if forced_durations is None else self._forced(forced_durations, sentences)
        self.control = [None] * self.S
        if duration_scale is not None:
            for i, ph in enumerate(sentences):
                sc = S.duration_control(duration_scale, None, None, B, ph.shape[1])
                if sc[0].dim() > 1:
                    raise L.MttsError(f"duration_scale: shape {tuple(sc[0].shape)}, expected () or ({B},) (per-phone "
                                      f"scales would differ per sentence)")
                self.control[i] = sc
        if sampling is not None and not isinstance(sampling, S.Sampling):
            raise L.MttsError(f"sampling must be a megatts2_b200.sampling.Sampling, got {type(sampling).__name__}")
        self.sampling = sampling
        self.keys = None if sampling is None else S.row_keys(keys, B, "cpu").tolist()
        self.sentences, self.mels = list(sentences), mels

    def _pauses(self, pause_frames):
        B, S_ = self.B, self.S
        if isinstance(pause_frames, (int, np.integer)) and not isinstance(pause_frames, bool):
            if pause_frames < 0:
                raise L.MttsError(f"pause_frames must be >= 0, got {pause_frames}")
            return [[int(pause_frames)] * (S_ - 1) for _ in range(B)]
        p = S._integers(pause_frames, "pause_frames", "(B, S - 1)")
        if tuple(p.shape) != (B, S_ - 1):
            raise L.MttsError(f"pause_frames: shape {tuple(p.shape)}, expected an int or ({B}, {S_ - 1})")
        if bool((p < 0).any()):
            b, i = (int(x) for x in (p < 0).nonzero()[0])
            raise L.MttsError(f"pause_frames[{b}, {i}] = {int(p[b, i])}: the pause after sentence {i} of row {b} must "
                              "be >= 0 frames")
        return p.tolist()

    def _context(self, plm_context, vq_bins, tc_dim):
        if plm_context is None:
            return None
        from .models.megatts2 import PLMContext
        c = PLMContext.cat(plm_context if isinstance(plm_context, (list, tuple)) else [plm_context])
        if c.tc8.shape[0] not in (1, self.B):
            raise L.MttsError(f"plm_context: Bc = {c.tc8.shape[0]}, expected 1 or B = {self.B}")
        if c.tc8.shape[2] != tc_dim or c.tc8.device != self.device:
            raise L.MttsError(f"plm_context: latents (Bc, P, {tc_dim}) on {self.device}, got {tuple(c.tc8.shape)} on "
                              f"{c.tc8.device}")
        if c.max_code >= vq_bins:
            raise L.MttsError(f"plm_context: codes must be in [0, {vq_bins}), got {c.max_code}")
        return c

    def _forced(self, forced, sentences):
        if isinstance(forced, torch.Tensor) or not isinstance(forced, (list, tuple)) or len(forced) != self.S:
            raise L.MttsError(f"forced_durations: expected a list of {self.S} (B, Tp_i) tensors, one per sentence")
        out = []
        for i, (fd, ph) in enumerate(zip(forced, sentences)):
            d = S._integers(fd, f"forced_durations[{i}]", "(B, Tp_i)")
            if tuple(d.shape) != tuple(ph.shape):
                raise L.MttsError(f"forced_durations[{i}]: shape {tuple(d.shape)}, expected {tuple(ph.shape)} "
                                  f"(sentences[{i}])")
            if bool((d < 0).any()):
                b, j = (int(x) for x in (d < 0).nonzero()[0])
                raise L.MttsError(f"forced_durations[{i}][{b}, {j}] = {int(d[b, j])}: durations must be >= 0")
            out.append(fd if isinstance(fd, torch.Tensor) and fd.device == self.device and fd.dtype == torch.int32
                       else d.to(torch.int32))
        return out


# ------------------------------------------------------------------------------ device side
class History:
    """The prosody LM's context history on the device: per row the last ``kept[b]`` rows of its history (at most
    ``context_rows``, or the initial context's P), in ``tc8`` (Bc, K, tc_dim) and ``codes`` (Bc, K), Bc = 1 or B.  ``H``
    counts every history row of each row.  Each join is one ``ops.copy_row_segments`` per tensor."""

    def __init__(self, B, context_rows, context):
        self.B, self.context_rows = B, context_rows
        if context is None:
            self.tc8 = self.codes = None
            self.kept, self.max_code = [0] * B, -1
        else:
            self.tc8, self.codes = context.tc8, context.codes
            self.kept, self.max_code = [context.P] * B, context.max_code
        self.H = list(self.kept)

    def window(self):
        """-> (W, P): the last P = min(context_rows, min_b H_b) rows of each row's history as a PLMContext with Bc = B
        (None when P = 0)."""
        from . import ops
        from .models.megatts2 import PLMContext
        B, P = self.B, window_rows(self.H, self.context_rows)
        if P == 0:
            return None, 0
        tc8 = torch.empty(B, P, self.tc8.shape[2], dtype=torch.float32, device=self.tc8.device)
        codes = torch.empty(B, P, dtype=torch.int64, device=self.tc8.device)
        off = [k - P for k in self.kept]
        ops.copy_row_segments(tc8, [0] * B, [P] * B, src=self.tc8, src_off=off)
        ops.copy_row_segments(codes, [0] * B, [P] * B, src=self.codes, src_off=off)
        return PLMContext.from_rows(tc8, codes, self.max_code), P

    def append(self, tc8, codes, totals, vq_bins):
        """Appends a sentence's valid rows (its ``tc8`` and ``codes`` (B, T8), ``totals`` frames per row)."""
        from . import ops
        if self.context_rows == 0:
            return
        B, n = self.B, codes_rows(totals)
        keep, o, m = history_update(self.kept, n, self.context_rows)
        K = max(keep)
        new_tc8 = torch.empty(B, K, tc8.shape[2], dtype=torch.float32, device=tc8.device)
        new_codes = torch.empty(B, K, dtype=torch.int64, device=tc8.device)
        if self.tc8 is not None and any(o):
            off = [k - ob for k, ob in zip(self.kept, o)]
            ops.copy_row_segments(new_tc8, [0] * B, o, src=self.tc8, src_off=off)
            ops.copy_row_segments(new_codes, [0] * B, o, src=self.codes, src_off=off)
        off = [nb - mb for nb, mb in zip(n, m)]
        ops.copy_row_segments(new_tc8, o, m, src=tc8, src_off=off)
        ops.copy_row_segments(new_codes, o, m, src=codes, src_off=off)
        self.tc8, self.codes, self.kept = new_tc8, new_codes, keep
        self.H = [h + nb for h, nb in zip(self.H, n)]
        self.max_code = max(self.max_code, vq_bins - 1)


class PassageMel:
    """Row b's passage mel, assembled sentence by sentence: ``place`` appends a sentence's frames and the pause after
    it (one ``ops.copy_row_segments`` each).  ``f[b]``: the frames placed in row b; rows past it are zero."""

    def __init__(self, B, mel_bins, device):
        self.buf = torch.zeros(B, 0, mel_bins, dtype=torch.float32, device=device)
        self.f = [0] * B

    def place(self, mel, totals, pause=None):
        from . import ops
        B = len(self.f)
        ends = [f + int(t) for f, t in zip(self.f, totals)]
        pause = pause or [0] * B
        need = max(e + p for e, p in zip(ends, pause))
        if need > self.buf.shape[1]:
            grown = torch.zeros(B, max(need, 2 * self.buf.shape[1]), self.buf.shape[2], dtype=torch.float32,
                                device=self.buf.device)
            grown[:, :self.buf.shape[1]] = self.buf
            self.buf = grown
        ops.copy_row_segments(self.buf, self.f, [int(t) for t in totals], src=mel, src_off=[0] * B)
        if any(pause):
            ops.copy_row_segments(self.buf, ends, pause, fill=SILENCE)
        self.f = [e + p for e, p in zip(ends, pause)]


def run_sentences(tts, plan, guard):
    """Sentence by sentence: ``Megatts._synthesize`` up to the mel decoder, with the window of the history before it,
    the sentence's keys, and the prompt encoded once.  Yields (the sentence's result, P_i) after the sentence entered
    the history.  With ``guard`` the range flag is read after the prompt's encoding and after each sentence; a raised
    flag redoes that piece on bf16x3.  The AR decodes run eagerly (``graphs.disabled()``): a passage's sentence shapes
    rarely repeat, and capturing them would evict the graphs the caller's own calls replay."""
    from . import graphs, ops, pack
    from .models.megatts2 import _warn_fp16_range
    dev, mrte = plan.device, tts.generator.mrte
    encodings = {}

    def encoding():
        e = pack.default_engine()
        if e not in encodings:
            encodings[e] = mrte.encode_prompt(plan.mels)
        return encodings[e]

    with graphs.disabled(), torch.no_grad():
        encoding()
        if guard and ops.tc_overflow(dev):
            _warn_fp16_range("encoding this passage's prompt on the bf16x3 engine")
            with pack.engine_scope(pack.ENGINE_BF16X3):
                encodings[pack.ENGINE_BF16X3] = mrte.encode_prompt(plan.mels)
            encodings = {e: encodings[pack.ENGINE_BF16X3] for e in (pack.default_engine(), pack.ENGINE_BF16X3)}
    hist = History(plan.B, plan.context_rows, plan.context)
    for i, ph in enumerate(plan.sentences):
        ctx, P = hist.window()
        keys = None if plan.sampling is None else torch.tensor(sentence_keys(plan.keys, i), dtype=torch.int64)
        forced = None if plan.forced is None else plan.forced[i]
        args = (ph, plan.mels, forced, False, None, None, plan.sampling, keys, None, None, None, ctx, plan.control[i])
        with graphs.disabled(), torch.no_grad():
            out = tts._synthesize(*args, mel_context=encoding(), mel_only=True)
            if guard and ops.tc_overflow(dev):
                _warn_fp16_range(f"re-running sentence {i} of this passage on the bf16x3 engine")
                with pack.engine_scope(pack.ENGINE_BF16X3):
                    out = tts._synthesize(*args, mel_context=encoding(), mel_only=True)
        if i < plan.S - 1:
            with torch.no_grad():
                hist.append(out["tc8"], out["p_codes"], out["totals"], tts.plm.vq_bins)
        yield out, P


def vocode(tts, mel, rows, lens, guard):
    """The vocoder over ``mel[rows, :n]`` for each group of the given rows with equal n = ``lens[k]`` (one launch
    sequence per group) -> {length n: (row index list, wav (len(rows_of_group), 1, 256 (n + 10)))}.  With ``guard`` the
    range flag is read after the launches, and a raised flag redoes them on bf16x3."""
    from . import ops, pack
    from .models.megatts2 import _warn_fp16_range
    groups = {}
    for r, n in zip(rows, lens):
        groups.setdefault(n, []).append(r)

    def run():
        out = {}
        for n, ids in groups.items():
            idx = torch.tensor(ids, device=mel.device)
            out[n] = ids, tts.hifi_gan.decode_batch_cl(mel[idx, :n] if len(ids) < mel.shape[0] else mel[:, :n])
        return out
    out = run()
    if guard and ops.tc_overflow(mel.device):
        _warn_fp16_range("re-running this passage's vocoder on the bf16x3 engine")
        with pack.engine_scope(pack.ENGINE_BF16X3):
            out = run()
    return out
