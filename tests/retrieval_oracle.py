"""NumPy restatement of K17's contract (merlot_rank_topk, include/merlot_b200.h) and of retrieval_validate's metrics, for
the host and GPU tests.  Written from the contract, not from the kernel: plain comparisons over whole rows and a stable sort."""
import numpy as np


def rank_topk(scores: np.ndarray, pos: np.ndarray, k: int):
    """scores fp32 [rows, cols], pos int [rows] -> (greater, ties, topk_idx, topk_val) as K17 defines them."""
    s = np.asarray(scores, np.float32)
    rows, cols = s.shape
    greater = np.zeros(rows, np.int32)
    ties = np.zeros(rows, np.int32)
    idx = np.full((rows, k), -1, np.int32)
    val = np.full((rows, k), np.nan, np.float32)
    for r in range(rows):
        row, p = s[r], int(pos[r])
        if not 0 <= p < cols:
            greater[r] = -2
        elif np.isnan(row[p]):
            greater[r] = -1
        else:
            greater[r] = int(np.sum(row > row[p]))
            ties[r] = int(np.sum(row == row[p])) - 1
        ok = np.flatnonzero(~np.isnan(row))
        order = ok[np.lexsort((ok, -row[ok].astype(np.float64)))][:k]  # score descending, then index ascending
        idx[r, :len(order)] = order
        val[r, :len(order)] = row[order]
    return greater, ties, idx, val


def cosine_ranks(q: np.ndarray, keys: np.ndarray):
    """float64 cosine scores of every query row against every key row, 1 + the number of keys scoring above the positive
    (query i's positive is key i), and each query's margin: the smallest distance between its positive's score and any other
    key's score."""
    qn = q / np.linalg.norm(q, axis=1, keepdims=True)
    kn = keys / np.linalg.norm(keys, axis=1, keepdims=True)
    s = qn.astype(np.float64) @ kn.astype(np.float64).T
    d = np.diag(s)
    rank = 1 + np.sum(s > d[:, None], axis=1)
    other = s.copy()
    np.fill_diagonal(other, -np.inf)
    gap = np.min(np.abs(other - d[:, None]), axis=1)
    return s, rank, gap
