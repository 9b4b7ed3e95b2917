"""Host restatement of long-form synthesis's bookkeeping (megatts2_b200/passage.py), written from the rules rather than
from the implementation: each row's whole history is kept as a list, and the window, the keys, the pause layout and
the frame offsets are read off it."""

FRAMES_PER_CODE = 8


def window(initial_rows, sentence_totals, context_rows):
    """The (P, [(source, index) per row]) window of the next sentence.  ``initial_rows``: the initial context's P0 (0
    without one); ``sentence_totals``: the frame totals [L_b] of each earlier sentence.  Row b's history is the list of
    its rows, ('ctx', j) for the context and (s, j) for row j of sentence s's max-pooled latents; the window is the last
    P = min(context_rows, min_b len(history_b)) entries of each."""
    B = len(sentence_totals[0]) if sentence_totals else None
    hist = None
    if B is None:
        return min(context_rows, initial_rows), None
    hist = [[("ctx", j) for j in range(initial_rows)] for _ in range(B)]
    for s, totals in enumerate(sentence_totals):
        for b, L in enumerate(totals):
            hist[b] += [(s, j) for j in range((L + FRAMES_PER_CODE - 1) // FRAMES_PER_CODE)]
    P = min([context_rows] + [len(h) for h in hist])
    return P, [h[len(h) - P:] for h in hist]


def key(k, i):
    """Sentence i's key for row key k: k + i * 2^32 as a wrapping int64."""
    v = (k + i * 2 ** 32) & (2 ** 64 - 1)
    return v - 2 ** 64 if v >= 2 ** 63 else v


def layout(totals, pauses):
    """The passage mel of each row as a list of ('s', i, j) (frame j of sentence i) and ('pause', i) entries, and the
    frame where each sentence starts -> (frames per row, offsets per row)."""
    S, B = len(totals), len(totals[0])
    frames, offsets = [], []
    for b in range(B):
        fr, off = [], []
        for i in range(S):
            off.append(len(fr))
            fr += [("s", i, j) for j in range(totals[i][b])]
            if i < S - 1:
                fr += [("pause", i)] * pauses[b][i]
        frames.append(fr)
        offsets.append(off)
    return frames, offsets
