"""Speech editing's host side (``Megatts.edit``): the validated edit of B utterances and the prosody-code pins that keep
the unedited frames' codes.

An edit replaces the original phones [a, b) of utterance row r by n new ones, so that ``phone_tokens`` is
``orig_phone[:a] + new + orig_phone[b:]``.  The kept phones keep their original durations (pins of the ADM loop) and
the new ones are decoded.  In mel frames, with d the original durations:

    F_a = sum d[:a] (the kept prefix), L_o = sum d[a:b] (the replaced frames), F_s = sum d[b:] (the kept suffix),
    L_n = the new phones' frames, N_e = F_a + L_n + F_s, s = L_n - L_o (the suffix's shift).

The prosody LM decodes one code per block of 8 frames.  Block k of the edited utterance is pinned to an original code
when it holds original frames only (``code_pins``): a full block of prefix frames keeps ``orig_codes[k]``; a block of
suffix frames, which are original frames shifted by s, keeps the code of the original block holding most of them (the
lower block on a tie, so ``orig_codes[k - s / 8]`` when 8 divides s); a block past the utterance's end, which the mel
decoder never reads, is pinned to 0.  The other blocks overlap the new frames or straddle one of their ends and are
decoded, so prosody edits are quantised to 8 frames."""
import torch

from . import _lib as L
from . import sampling as S

FRAMES_PER_CODE = 8
# arguments of ``synthesize`` that an edit sets itself or does not support
REJECTED = ("forced_durations", "causal_decode", "pinned_durations", "total_frames", "prompt_mels", "prosody_mels",
            "prosody_weights", "duration_weights", "timbre_mels", "timbre_weights")


def _ints(v, what, dims):
    t = S._integers(v, what, dims)
    if t.dim() != len([x for x in dims.strip("()").split(",") if x.strip()]):
        raise L.MttsError(f"{what}: expected a {dims} array, got shape {tuple(t.shape)}")
    return t


class EditPlan:
    """A validated edit (every check on the host, before any device work): the row-wise prefix / replaced / suffix
    frame counts, the ADM pins and target totals of ``synthesize``'s duration control, and the rule for the code pins.
    Each error names the row and, where there is one, the position."""

    def __init__(self, phone_tokens, orig_phone, orig_durations, orig_codes, span, span_frames, vq_bins):
        ph, oph = _ints(phone_tokens, "phone_tokens", "(B, Tp_e)"), _ints(orig_phone, "orig_phone", "(B, Tp_o)")
        d = _ints(orig_durations, "orig_durations", "(B, Tp_o)")
        codes = _ints(orig_codes, "orig_codes", "(B, T_o)")
        sp = _ints(span, "span", "(B, 2)")
        B, Tp_e = ph.shape
        Tp_o = oph.shape[1]
        if oph.shape[0] != B or tuple(d.shape) != (B, Tp_o) or codes.shape[0] != B or tuple(sp.shape) != (B, 2):
            raise L.MttsError(f"edit: expected orig_phone and orig_durations (B, Tp_o), orig_codes (B, T_o) and span "
                              f"(B, 2) with B = {B}, got {tuple(oph.shape)}, {tuple(d.shape)}, {tuple(codes.shape)} and "
                              f"{tuple(sp.shape)}")
        sf = None if span_frames is None else _ints(span_frames, "span_frames", "(B,)")
        if sf is not None and tuple(sf.shape) != (B,):
            raise L.MttsError(f"span_frames: shape {tuple(sf.shape)}, expected ({B},)")
        self.B, self.Tp_e, self.Tp_o = B, Tp_e, Tp_o
        phl, ophl, dl, spl = ph.tolist(), oph.tolist(), d.tolist(), sp.tolist()
        sfl = None if sf is None else sf.tolist()
        self.a, self.b, self.n, self.F_a, self.L_o, self.F_s = [], [], [], [], [], []
        pins = torch.full((B, Tp_e), -1, dtype=torch.int32)
        for r in range(B):
            a, b = spl[r]
            if not 0 <= a <= b <= Tp_o:
                raise L.MttsError(f"span[{r}] = [{a}, {b}): expected 0 <= a <= b <= Tp_o = {Tp_o}")
            n = Tp_e - Tp_o + (b - a)
            if n < 0:
                raise L.MttsError(f"span[{r}] = [{a}, {b}): phone_tokens has {Tp_e} phones, {-n} fewer than the "
                                  f"{Tp_o - (b - a)} the edit keeps")
            for j in range(a):
                if phl[r][j] != ophl[r][j]:
                    raise L.MttsError(f"phone_tokens[{r}, {j}] = {phl[r][j]} differs from orig_phone[{r}, {j}] = "
                                      f"{ophl[r][j]} before the span")
            for j in range(b, Tp_o):
                je = j - b + a + n
                if phl[r][je] != ophl[r][j]:
                    raise L.MttsError(f"phone_tokens[{r}, {je}] = {phl[r][je]} differs from orig_phone[{r}, {j}] = "
                                      f"{ophl[r][j]} after the span")
            for j in range(Tp_o):
                v = dl[r][j]
                if (j < a or j >= b) and not 1 <= v <= S.PIN_MAX:
                    raise L.MttsError(f"orig_durations[{r}, {j}] = {v}: a kept phone's duration must be in "
                                      f"1..{S.PIN_MAX} (the ADM's pin range)")
                if v < 0:
                    raise L.MttsError(f"orig_durations[{r}, {j}] = {v}: durations must be >= 0")
            F_a, L_o, F_s = sum(dl[r][:a]), sum(dl[r][a:b]), sum(dl[r][b:])
            need = -(-(F_a + L_o + F_s) // FRAMES_PER_CODE)
            if codes.shape[1] < need:
                raise L.MttsError(f"orig_codes[{r}]: {codes.shape[1]} codes, but its {F_a + L_o + F_s} frames need "
                                  f"{need}")
            row = codes[r, :need]
            if need and (int(row.min()) < 0 or int(row.max()) >= vq_bins):
                j = int(((row < 0) | (row >= vq_bins)).nonzero()[0])
                raise L.MttsError(f"orig_codes[{r}, {j}] = {int(row[j])}: expected 0..{vq_bins - 1}")
            if sfl is not None and not n <= sfl[r] <= S.DURATION_MAX * n:
                raise L.MttsError(f"span_frames[{r}] = {sfl[r]}: the {n} new phones of row {r} take "
                                  f"{n} to {S.DURATION_MAX * n} frames")
            pins[r, :a] = d[r, :a].to(torch.int32)
            pins[r, a + n:] = d[r, b:].to(torch.int32)
            for lst, v in ((self.a, a), (self.b, b), (self.n, n), (self.F_a, F_a), (self.L_o, L_o), (self.F_s, F_s)):
                lst.append(v)
        self.pinned_durations = pins
        self.total_frames = None if sf is None else torch.tensor(
            [self.F_a[r] + sfl[r] + self.F_s[r] for r in range(B)], dtype=torch.int64)
        self.orig_codes = codes.tolist()

    def new_frames(self, totals):
        """The new phones' frame counts L_n per row, from the edited utterances' frame totals N_e."""
        return [int(totals[r]) - self.F_a[r] - self.F_s[r] for r in range(self.B)]

    def edit_frames(self, totals):
        """(B, 2) int64: [F_a, F_a + L_n), the regenerated frames of each edited utterance."""
        L_n = self.new_frames(totals)
        return torch.tensor([[self.F_a[r], self.F_a[r] + L_n[r]] for r in range(self.B)], dtype=torch.int64)

    def code_pins(self, totals, T):
        """(B, T) int32 code pins of the edited utterances whose frame totals are ``totals``: -1 for a decoded block,
        else the original code it keeps (0 past the utterance's end; the module docstring states the rule)."""
        L_n = self.new_frames(totals)
        rows = [[-1] * T for _ in range(self.B)]
        for r in range(self.B):
            F_a, N_e, orig, pr = self.F_a[r], int(totals[r]), self.orig_codes[r], rows[r]
            s = L_n[r] - self.L_o[r]
            for k in range(T):
                lo, hi = FRAMES_PER_CODE * k, min(FRAMES_PER_CODE * (k + 1), N_e)
                if lo + FRAMES_PER_CODE <= F_a:
                    pr[k] = orig[k]
                elif lo >= N_e:
                    pr[k] = 0
                elif lo >= F_a + L_n[r]:
                    g0, g1 = lo - s, hi - s                            # the original frames of the block
                    q = g0 // FRAMES_PER_CODE
                    c0 = min(FRAMES_PER_CODE * (q + 1), g1) - g0       # in original block q; the rest in q + 1
                    pr[k] = orig[q if c0 >= g1 - g0 - c0 else q + 1]
        return torch.tensor(rows, dtype=torch.int32).reshape(self.B, T)
