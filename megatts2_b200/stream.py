"""Chunk schedule of ``Megatts.synthesize_stream``: pure host arithmetic, no device work.

Positions count mel frames of the padded waveform ``synthesize`` returns (without the prompt): position p is sample
``hop * p``, mel frame f owns positions [f + pad, f + pad + 1), and the vocoder's ``pad`` replicated frames put positions
[0, pad) before frame 0 and [L + pad, L + 2 pad) after the last.  Chunk k of a stream whose longest utterance has
``L_total`` frames covers positions [P_k, P_k+1) with P_0 = 0, P_k = k * chunk_frames + pad and P_K = L_total + 2 pad, so
the first chunk carries the leading pad and the last the trailing pad.

For one utterance of L frames, the samples of positions [p0, p1) depend on frames [p0 - pad - hv, p1 - pad + hv) clipped
to [0, L) (hv: the vocoder's receptive field); those frames' mel rows depend on decoder inputs hd frames further out, and
a mel row f on code f // 8.  Window starts are aligned down to a multiple of 8 so that the x8 code repeat of the decoder
input lines up; a window edge is either the sequence's edge or at least a halo away from every row it produces."""
import dataclasses


@dataclasses.dataclass(frozen=True)
class Chunk:
    p0: int            # positions [p0, p1) of the waveform: samples [hop * p0, hop * p1)
    p1: int
    a: int             # mel frames [a, b) whose own positions lie in [p0, p1)
    b: int
    rows: tuple        # (r0, r1): mel rows decoded for this chunk (r0 == r1: none)
    dec: tuple         # (da, db): decoder window producing those rows (None when no rows are decoded)
    voc: tuple         # (va, vb): vocoder window
    t1: int            # PLM steps that must be decoded before this chunk: codes [0, t1)


def _down8(x):
    return x - x % 8


def chunk_positions(L_total, chunk_frames, pad):
    """[P_0, ..., P_K]: the chunk boundaries of a stream whose longest utterance has L_total >= 1 frames."""
    if L_total < 1 or chunk_frames < 1:
        raise ValueError(f"chunk_positions: need L_total >= 1 and chunk_frames >= 1, got {L_total}, {chunk_frames}")
    K = -(-L_total // chunk_frames)
    return [0] + [k * chunk_frames + pad for k in range(1, K)] + [L_total + 2 * pad]


def schedule(L, chunk_frames, hd, hv, pad, L_total=None):
    """The chunks of one utterance of L frames in a stream whose longest utterance has L_total >= L frames (default L):
    one entry per chunk of that stream, None where the utterance has no samples (past its end)."""
    L_total = L if L_total is None else L_total
    if not 0 <= L <= L_total:
        raise ValueError(f"schedule: need 0 <= L <= L_total, got {L}, {L_total}")
    P = chunk_positions(L_total, chunk_frames, pad)
    out, done, t1 = [], 0, 0                     # done: mel rows [0, done) decoded by earlier chunks
    for k in range(len(P) - 1):
        p0, p1 = P[k], min(P[k + 1], L + 2 * pad)
        if L == 0 or p0 >= p1:
            out.append(None)
            continue
        a, b = min(max(p0 - pad, 0), L), min(max(p1 - pad, 0), L)
        va = _down8(min(max(p0 - pad - hv, 0), L - 1))
        vb = min(max(p1 - pad + hv, va + 1), L)
        if vb > done:
            rows = (done, vb)
            dec = (_down8(max(done - hd, 0)), min(vb + hd, L))
            t1 = max(t1, -(-dec[1] // 8))
            done = vb
        else:
            rows, dec = (done, done), None
        out.append(Chunk(p0, p1, a, b, rows, dec, (va, vb), t1))
    return out
