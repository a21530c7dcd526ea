"""ctypes bindings of oracle/oracle_emdepth.c, a literal restatement of emdepth.Cache (emdepth/emdepth.go:306-398) and the
`goleft emdepth` driver and text — TEST INFRASTRUCTURE ONLY (same rules as oracle/loader.py)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle.dcnv import Panic, _WS, _atof, _atoi
from oracle.loader import _proto, _ptr, _vp, lib

_proto("orc_em_factors", None, _vp)
_proto("orc_emdepth", C.c_int, _vp, C.c_int64, C.c_int64, C.c_int, _vp, _vp, _vp)

M32 = 0xFFFFFFFF
LOWER, UPPER = -0.80, 0.40


def factors() -> np.ndarray:
    f = np.empty(9, np.float64)
    lib.orc_em_factors(_ptr(f))
    return f


def emdepth(x):
    """EMDepth + CN + Log2FC of every row of the n x S float32 matrix x -> (cells uint8 n x S, lambda n x 9, fc n x S)"""
    x = np.ascontiguousarray(x, np.float32)
    if x.ndim == 1:
        x = x[None, :]
    n, S = x.shape
    cells, lam, fc = np.empty((n, S), np.uint8), np.empty((n, 9), np.float64), np.empty((n, S), np.float64)
    rc = lib.orc_emdepth(_ptr(x), n, S, S, _ptr(cells), _ptr(lam), _ptr(fc))
    if rc == -1:
        raise Panic("%d samples: median32 indexes out of range" % S)
    if rc < -1:
        raise Panic("row %d has a value the library rejects" % (-2 - rc))
    return cells, lam, fc


# 2^-0.8 as the library compares Log2FC's lower Same threshold in ratio space
Q_M08 = 0.57434917749851755


def near_tie_rows(want: int, count: int = 1000, V: float = 100.0) -> np.ndarray:
    """Rows of count + 1 float32 values whose Log2FC for the middle sample lies within 4e-13 (relative, in ratio space) of
    -0.8: count values at V plus K float32 steps between them (bin 2, whose exact mean is lambda[2]) and one d in bin 1
    with d / lambda[2] = 2^-0.8 (1 + 4e-13).  Found by walking d upwards one float32 step at a time and choosing K."""
    ulp = 2.0 ** -17                                                    # float32 spacing in [64, 128)
    d, out = np.float32(Q_M08 * V), []
    while len(out) < want:
        d = np.nextafter(d, np.float32(128), dtype=np.float32)
        K = round((float(d) / Q_M08 - V) * count / ulp)
        l2 = (count * V + K * ulp) / count                              # the bin-2 sum is exact; one rounding in the division
        if abs(float(d) / l2 / Q_M08 - 1) < 4e-13:
            base, extra = divmod(K, count)
            xs = np.full(count, V + base * ulp)
            xs[:extra] += ulp
            out.append(np.concatenate([xs[:count // 2], [float(d)], xs[count // 2:]]).astype(np.float32))
    return np.array(out)


def cns(x) -> list:
    return [int(c) & 15 for c in emdepth(x)[0][0]]


class EMD:
    def __init__(self, fc, cn, pos, row=None):
        self.fc, self.cn, self.pos, self.row = fc, cn, pos, row


def same(e: EMD, o: EMD):
    """e.Same(o) -> (non2, changed, pct)"""
    non2, changed, n_same = [], [], 0.0
    for i, ee in enumerate(e.fc):
        oo = o.fc[i]
        if LOWER < ee < UPPER and LOWER < oo < UPPER:
            n_same += 1
            continue
        if (oo >= UPPER and ee >= UPPER) or (oo <= LOWER and ee <= LOWER):
            non2.append(i)
            n_same += 1
        else:
            changed.append(i)
    return non2, changed, n_same / len(e.fc)


def makecnvs(es, sample):
    cnv = None
    for e in es:
        fc = e.fc[sample]
        if -0.5 < fc < 0.3:
            continue
        if cnv is None:
            cnv = dict(sample=sample, cn=[e.cn[sample]], pos=[e.pos], rows=[e.row])
            continue
        cnv["cn"].append(e.cn[sample])
        cnv["pos"].append(e.pos)
        cnv["rows"].append(e.row)
    return cnv


class Cache:
    """emdepth.Cache; its map is a dict, walked in sample order (Go's order is random)"""

    def __init__(self):
        self.last, self.cnvs = None, None

    def add(self, e: EMD):
        if self.last is None:
            if self.cnvs is None:
                self.cnvs = {}
            self.last = e
        ret = self.clear(e.pos)
        non2, _, _ = same(self.last, e)
        for si in non2:
            self.cnvs.setdefault(si, []).append(e)
        self.last = e
        return ret

    def clear(self, p):
        if p is None:
            if self.last is None:
                return []
            p = ((self.last.pos[0] + 100000) & M32, (self.last.pos[1] + 100000) & M32)
        out = []
        keys = [0] * len(self.cnvs)                                      # make([]int, len(c.cnvs))
        for si in sorted(self.cnvs):
            emd = self.cnvs[si]
            if (p[0] - emd[-1].pos[1]) & M32 < 30000:
                continue
            put = makecnvs(emd, si)
            if put is not None:
                put["psize"] = len(self.cnvs)
                out.append(put)
                keys.append(si)
        for k in keys:
            self.cnvs.pop(k, None)
        return out


def drive(chroms, starts, ends, fc, cn):
    """The driver: one Cache over the rows in order, Clear(nil) at every chromosome change and at the end -> CNVs, each with
    its first row's chromosome"""
    c, out = Cache(), []
    for r in range(len(starts)):
        if r > 0 and chroms[r] != chroms[r - 1]:
            out += c.clear(None)
        out += c.add(EMD(fc[r], cn[r], (int(starts[r]), int(ends[r])), r))
    out += c.clear(None)
    return out


def read_matrix(text: bytes):
    """dcnv's matrix rules without the 250 clamp -> (header fields, chroms, starts, ends, x float64 n x S)"""
    header, chroms, starts, ends, vals, i = None, [], [], [], [], 0
    for ln in text.split(b"\n")[:-1]:                                   # a final line without "\n" is dropped
        line = ln + b"\n"
        if i == 0 and (line[:1] == b"#" or line.startswith(b"chrom")):
            f = line.strip(_WS).split(b"\t")
            if len(f) < 3:
                raise Panic("header has fewer than 3 fields")
            header = f
            continue
        i += 1
        toks = line.split(b"\t")
        toks[-1] = toks[-1].strip(_WS)
        if len(toks) < 3:
            raise Panic("fewer than 3 columns")
        s, e = _atoi(toks[1]), _atoi(toks[2])
        ns = len(header) - 3 if header is not None else 0
        if len(toks) - 3 != ns:
            raise Panic("row has %d values, header has %d samples" % (len(toks) - 3, ns))
        chroms.append(toks[0]); starts.append(s); ends.append(e)
        vals.append([_atof(t) for t in toks[3:]])
    if header is None or len(header) == 3:
        raise Panic("no samples")
    S = len(header) - 3
    return header, chroms, starts, ends, np.asarray(vals, np.float64).reshape(len(vals), S)


def files(text: bytes):
    """(P.cn.bed, P.cnv.bed) bytes of `goleft emdepth` on a matrix"""
    header, chroms, starts, ends, x = read_matrix(text)
    S = x.shape[1]
    if S == 2:
        raise Panic("2 samples: median32 indexes out of range")
    cells, _, fc = emdepth(x.astype(np.float32)) if len(starts) else (np.empty((0, S), np.uint8), None, np.empty((0, S)))
    cn = (cells & 15).astype(int)
    cn_bed = [b"\t".join(header)]
    for r in range(len(starts)):
        cn_bed.append(b"%s\t%d\t%d\t" % (chroms[r], starts[r], ends[r]) + b"\t".join(b"%d" % v for v in cn[r]))
    cnv_bed = [b"#chrom\tstart\tend\tsample\tn\tcns\tpsize"]
    for v in drive(chroms, starts, ends, fc, cn):
        cnv_bed.append(b"%s\t%d\t%d\t%s\t%d\t%s\t%d" % (chroms[v["rows"][0]], v["pos"][0][0], v["pos"][-1][1], header[3 + v["sample"]],
                                                        len(v["cn"]), b",".join(b"%d" % c for c in v["cn"]), v["psize"]))
    return b"\n".join(cn_bed) + b"\n", b"\n".join(cnv_bed) + b"\n"
