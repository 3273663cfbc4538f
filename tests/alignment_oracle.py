"""CPU oracle of token timestamps: openai-whisper's median filter and DTW restated in numpy (the definitions transformers'
generation_whisper._median_filter / _dynamic_time_warping run), on one utterance's alignment x [frames, tokens]."""
import numpy as np


def median_filter(x: np.ndarray, width: int = 7) -> np.ndarray:
    """Median of `width` along frames (axis 0) with reflect padding; a matrix of width // 2 frames or fewer is returned as is."""
    half = width // 2
    F = x.shape[0]
    if F <= half:
        return x.copy()
    idx = np.arange(-half, F + half)
    idx = np.where(idx < 0, -idx, np.where(idx >= F, 2 * (F - 1) - idx, idx))
    win = np.stack([x[idx[k:k + F]] for k in range(width)], axis=0)   # [width, F, P]
    return np.sort(win, axis=0)[half]


def dtw_jumps(x: np.ndarray) -> np.ndarray:
    """The DTW of -x ([frames, tokens]) with fp32 cumulative costs and the tie order diagonal, previous token, previous frame;
    returns, per token, the first frame on the path."""
    F, P = x.shape
    cost = np.full((P + 1, F + 1), np.inf, dtype=np.float32)
    trace = np.full((P + 1, F + 1), -1, dtype=np.int8)
    cost[0, 0] = 0
    m = (-x.T).astype(np.float32)
    for j in range(1, F + 1):
        for i in range(1, P + 1):
            c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
            if c0 < c1 and c0 < c2:
                c, t = c0, 0
            elif c1 < c0 and c1 < c2:
                c, t = c1, 1
            else:
                c, t = c2, 2
            cost[i, j] = np.float32(m[i - 1, j - 1] + c)
            trace[i, j] = t
    first = np.zeros(P, dtype=np.int32)
    i, j = P, F
    while i > 0 or j > 0:
        if i > 0:
            first[i - 1] = j - 1
        t = 2 if i == 0 else (1 if j == 0 else trace[i, j])
        if t == 0:
            i, j = i - 1, j - 1
        elif t == 1:
            i -= 1
        else:
            j -= 1
    return first


def token_jumps(x: np.ndarray, key_mask=None, width: int = 7):
    """Filtered matrix and per-token first frames of one utterance; masked tokens (key_mask == 0) are dropped before the DTW
    and get -1."""
    filt = median_filter(x, width)
    P = x.shape[1]
    keep = np.ones(P, dtype=bool) if key_mask is None else np.asarray(key_mask) != 0
    jumps = np.full(P, -1, dtype=np.int32)
    if keep.any():
        jumps[keep] = dtw_jumps(filt[:, keep]) if x.shape[0] > 0 else 0
    return filt, jumps
