"""Slot vectors of a baby-step giant-step (BSGS) slot-wise linear transform, for B200Context.linear_transform.

With batching, a ciphertext holds a 2 x n/2 matrix of slots, and rotate_rows(s) rotates both rows left by s.  A d x d matrix M
(d divides n/2) applied to a vector v replicated with period d along a row is the diagonal method

    M v = sum_{i < d} diag_i(M) * rot_i(v),        diag_i[s] = M[s mod d][(s + i) mod d]

and in BSGS form, with i = g b + j and rot_i = rot_{g b} rot_j,

    M v = sum_g rot_{g b}( sum_j P[g][j] * rot_j(v) ),    P[g][j] = rot_{-g b}(diag_{g b + j}).

Each row of the slot matrix may carry its own matrix.  Transforms that mix the two rows need column rotations and are not
covered.
"""
import numpy as np


def bsgs_plain_vectors(mats, n, t, baby, giant=None):
    """mats: one d x d matrix for both slot rows, or a pair (row 0, row 1) of d x d matrices, d dividing n/2.
    Returns (vecs, present, steps):
      vecs     uint64 [giant][baby][n] slot vectors mod t (row 0 in [0, n/2), row 1 in [n/2, n)), to batch-encode;
      present  bool [giant][baby]: False where a diagonal is zero in both rows or g b + j >= d (an absent term);
      steps    the rotate_rows steps 1 .. baby - 1 then b, 2 b, .., (giant - 1) b: the Galois keys the transform needs.
    giant defaults to ceil(d / baby)."""
    if isinstance(mats, (list, tuple)) and len(mats) == 2 and np.ndim(mats[0]) == 2:
        rows = [np.asarray(m, dtype=object) for m in mats]
    else:
        rows = [np.asarray(mats, dtype=object)] * 2
    h = n // 2
    d = rows[0].shape[0]
    for m in rows:
        if m.shape != (d, d) or h % d:
            raise ValueError("each matrix must be d x d with d dividing n/2")
    if giant is None:
        giant = -(-d // baby)
    if baby * giant < d:
        raise ValueError("baby * giant must cover the d diagonals")
    s = np.arange(h)
    vecs = np.zeros((giant, baby, n), dtype=np.uint64)
    present = np.zeros((giant, baby), dtype=bool)
    for g in range(giant):
        for j in range(baby):
            i = g * baby + j
            if i >= d:
                continue
            for r, m in enumerate(rows):
                diag = np.array([int(m[x % d][(x + i) % d]) % t for x in range(h)], dtype=np.uint64)
                # rot_{-g b}: slot x takes diag[(x - g b) mod n/2]
                vecs[g, j, r * h:(r + 1) * h] = diag[(s - g * baby) % h]
            present[g, j] = bool(vecs[g, j].any())
    steps = list(range(1, baby)) + [g * baby for g in range(1, giant)]
    return vecs, present, steps


def apply_slotwise(mats, v, n, t):
    """The plain result the transform decrypts to: each slot row of v (length n) times its matrix, mod t, the row's vector
    taken with period d."""
    if isinstance(mats, (list, tuple)) and len(mats) == 2 and np.ndim(mats[0]) == 2:
        rows = [np.asarray(m, dtype=object) for m in mats]
    else:
        rows = [np.asarray(mats, dtype=object)] * 2
    h = n // 2
    out = np.zeros(n, dtype=np.uint64)
    for r, m in enumerate(rows):
        d = m.shape[0]
        x = np.asarray(v[r * h:r * h + d], dtype=object)
        y = m.dot(x) % t
        out[r * h:(r + 1) * h] = np.array([int(y[i % d]) for i in range(h)], dtype=np.uint64)
    return out
