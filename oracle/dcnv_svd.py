"""`goleft dcnv --svd PCT` restated in numpy float64 (DESIGN §1.13) — TEST INFRASTRUCTURE ONLY.

An independent route: the z-score with ddof=1 and the same exclusion of constant rows, then np.linalg.svd of Z itself (not
of the Gram), the same rank rule (sigma^2 <= 1e-12 sigma_1^2 counts as 0), the same count rule, Z - U_n S_n V_n^T, and
ZScore.UnScale (max(0, z sd + m))."""
from __future__ import annotations

import numpy as np

from oracle import dcnv as od

MAX_REMOVE = 15
RANK_TOL = 1e-12


def zscore(x):
    """(Z of the kept rows, kept mask, m, sd): a row whose values are all equal (every row when S < 2) is excluded"""
    x = np.asarray(x, np.float64)
    S = x.shape[1]
    kept = (x != x[:, :1]).any(axis=1) if S >= 2 else np.zeros(x.shape[0], bool)
    xk = x[kept]
    if not xk.shape[0]:
        return xk, kept, np.zeros(0), np.zeros(0)
    m = xk.mean(axis=1)
    sd = xk.std(axis=1, ddof=1)
    return (xk - m[:, None]) / sd[:, None], kept, m, sd


def singular_values(z, S: int) -> np.ndarray:
    """S values, descending, with the rank rule applied"""
    s = np.zeros(S)
    if z.shape[0]:
        sv = np.linalg.svd(z, compute_uv=False)
        s[:sv.size] = sv
    if s[0] > 0:
        s[s * s <= RANK_TOL * s[0] * s[0]] = 0
    else:
        s[:] = 0
    return s


def count(s, pct: float) -> int:
    """the reference's loop (debiaser.go:185), with its read past the values closed off: stop at min(15, rank)"""
    rank = int((np.asarray(s) > 0).sum())
    total = 0.0
    for v in s[:rank]:
        total += v
    n = 0
    while n < min(MAX_REMOVE, rank) and 100 * s[n] / total > pct:
        n += 1
    return n


def variance_text(s, n: int) -> bytes:
    total = 0.0
    for v in s[:int((np.asarray(s) > 0).sum())]:
        total += v
    return b"variance:" + b"".join(b" %.2f" % (100 * s[i] / total) for i in range(n))


def svd_debias(x, pct: float):
    """-> (result, singular values[S], n removed, kept mask)"""
    x = np.array(x, np.float64)
    S = x.shape[1]
    z, kept, m, sd = zscore(x)
    s = singular_values(z, S)
    n = count(s, pct)
    if n == 0:
        return x, s, 0, kept
    U, sv, Vt = np.linalg.svd(z, full_matrices=False)
    z2 = z - (U[:, :n] * sv[:n]) @ Vt[:n]
    x[kept] = np.maximum(0.0, z2 * sd[:, None] + m[:, None])
    return x, s, n, kept


def dcnv(text: bytes, fasta: bytes, fai: str, pct: float):
    """(depth.bed bytes, the values before "%.2f", the log line's text) of `dcnv --svd pct`"""
    samples, label, starts, ends, gc, x = od.read_regions(text, fasta, od.parse_fai(fai))
    out, _, _ = od.matrix(x, gc)
    res, s, n, _ = svd_debias(out, pct)
    body = b"#chrom\tstart\tend\t" + b"\t".join(samples) + b"\n" + od.rows(label, starts, ends, res)
    return body, res, variance_text(s, n)
