"""Relative-position bias in LUT form for the attention kernel.

Every ONE-PEACE bias table entry is ``rel_pos_table[rp_bucket[i, j]]`` where, away from the CLS row / column, the
bucket depends only on a per-position code difference: ``i - j`` for text / audio (adapter/text.py:18-29,
adapter/audio.py:20-32) and the 2-D offset ``(dh, dw)`` for images (adapter/image.py:19-34), with three extra ids for
the CLS row, CLS column and corner (text.py:64-68, image.py:30-33).  We therefore store, per head, a 1-D LUT such that

    bias[h][i][j] == lut[h][code_row[i] - code_col[j]]            for all 0 <= i, j < S

by giving CLS its own constant LUT regions (code_row[0] / code_col[0] are offset so that the difference lands there).
``build_lut_index`` derives the (bucket-id) LUT and the code arrays from the integer bucket matrix itself and verifies
the identity exhaustively, so a bucket scheme that is not of this form is detected (the caller then uses the dense
table with the mma.sync kernel).
"""
import numpy as np
import torch


def text_codes(S):
    """positions 1..S-1 -> code = position (bucket depends on i - j)."""
    return np.arange(S, dtype=np.int64)


def image_codes(S, w):
    """patch p = i - 1 at (p // w, p % w) -> code = (p // w) * (2w - 1) + p % w, so that code_i - code_j encodes (dh, dw)."""
    c = np.zeros(S, dtype=np.int64)
    p = np.arange(S - 1)
    c[1:] = (p // w) * (2 * w - 1) + (p % w)
    return c


def build_lut_index(bucket, codes):
    """bucket: int64 [S,S] numpy (bucket ids), codes: int64 [S] (codes[0] ignored).
    Returns (lut_idx int32 [L], code_row int32 [S], code_col int32 [S]) or None if the scheme is not a code-difference one."""
    S = bucket.shape[0]
    if S == 1:
        return np.array([bucket[0, 0]] * 4, dtype=np.int32), np.zeros(4, np.int32), np.zeros(4, np.int32)
    c = codes.astype(np.int64)
    maxc = int(c[1:].max())
    R1 = 2 * maxc + 1                 # CLS-row region  [R1, R1 + maxc]
    R2 = R1 + maxc + 1                # CLS-col region  [R2, R2 + 2 maxc]
    R3 = R1 + maxc + R2               # corner
    L = R3 + 1
    lut_idx = np.zeros(L, dtype=np.int64)
    diff = c[1:, None] - c[None, 1:] + maxc
    lut_idx[diff.reshape(-1)] = bucket[1:, 1:].reshape(-1)
    lut_idx[R1:R1 + maxc + 1] = bucket[0, 1]
    lut_idx[R2:R2 + 2 * maxc + 1] = bucket[1, 0]
    lut_idx[R3] = bucket[0, 0]
    code_row = c + maxc
    code_row[0] = R1 + maxc
    code_col = c.copy()
    code_col[0] = -R2
    # exhaustive check of the identity on bucket ids
    rebuilt = lut_idx[code_row[:, None] - code_col[None, :]]
    if not np.array_equal(rebuilt, bucket):
        return None
    # the kernel bulk-copies the LUT row and the column codes: lengths padded to 16-byte multiples
    pad4 = lambda a: np.concatenate([a, np.zeros((-a.size) % 4, dtype=a.dtype)])
    return pad4(lut_idx.astype(np.int32)), pad4(code_row.astype(np.int32)), pad4(code_col.astype(np.int32))


class LutCache:
    """Per-adapter cache: S -> device (lut_idx, code_row, code_col) or None when the LUT form does not apply."""

    def __init__(self):
        self._c = {}

    def get(self, S, device, bucket_tensor, codes_fn):
        key = (S, str(device))
        if key not in self._c:
            b = bucket_tensor[:S, :S].detach().cpu().numpy()
            r = build_lut_index(b, codes_fn(S))      # any length: a LUT too long to stage is read from global memory
            self._c[key] = None if r is None else tuple(torch.from_numpy(a).to(device) for a in r)
        return self._c[key]


def grid_codes(side):
    """Row-major side x side grid without a CLS row -> code = y * (2 side - 1) + x, so that code_i - code_j encodes (dy, dx)."""
    p = np.arange(side * side, dtype=np.int64)
    return (p // side) * (2 * side - 1) + p % side


def grid_lut_index(side, order=None):
    """LUT form of the bucket matrix ``make_image_bucket_position(side, ...)[1:, 1:]`` (the detection backbone's
    ``rp_bucket`` / ``rp_bucket_window``): bucket[i][j] = code_i - code_j + maxc with maxc = (side - 1) * 2 side, so
    lut_idx is the identity over the (2 side - 1)^2 table rows.  `order` (int64 [S'], row -> grid position) lays the codes
    out in another row order, e.g. window-major.  Returns (lut_idx, code_row, code_col) int32 numpy, lengths padded to 4."""
    c = grid_codes(side)
    if order is not None:
        c = c[np.asarray(order)]
    maxc = (side - 1) * 2 * side
    pad4 = lambda a: np.concatenate([a, np.zeros((-a.size) % 4, dtype=a.dtype)]).astype(np.int32)
    return pad4(np.arange((2 * side - 1) ** 2, dtype=np.int64)), pad4(c + maxc), pad4(c)


def window_major_order(side, window):
    """Row order that keeps every window x window window of a row-major side x side grid contiguous, windows row-major
    (detectron2's window_partition order).  Returns (perm int64 [side^2]: new row -> row-major position, y, x int64 [side^2]:
    global grid coordinates of each new row, ly, lx: coordinates inside its window)."""
    n = side // window
    wy, wx, ly, lx = np.meshgrid(np.arange(n), np.arange(n), np.arange(window), np.arange(window), indexing="ij")
    y, x = (wy * window + ly).reshape(-1), (wx * window + lx).reshape(-1)
    return y * side + x, y, x, ly.reshape(-1), lx.reshape(-1)
