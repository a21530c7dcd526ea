"""What `goleft indexcov` must write for a cohort of .bai files, derived from the oracle (oracle/loader.py for the depths,
rows, .roc and .ped bins, oracle/indexcov_pca.py for the PC columns).  The CLI tests of every cohort size share this one
derivation, so a small cohort and a large one are held to the same expectations."""
import os

import numpy as np

from bamutil import make_bai
from oracle import indexcov_pca as op
from oracle import loader as orc

COHORT_REFS = [("1", 3_000_000), ("2", 2_000_000), ("GL000207.1", 4262), ("X", 1_500_000), ("Y", 600_000), ("NC_007605", 171823)]


def cohort_bais(tmp_path, S=7, seed=3):
    """S .bai files over COHORT_REFS: even samples male (half X, half Y), odd female; sample 3 is 5 tiles short on "2".
    Returns (refs, fai path, bai paths, per-sample linear indexes)."""
    rng = np.random.default_rng(seed)
    refs = COHORT_REFS
    fai = tmp_path / "g.fa.fai"
    fai.write_text("".join("%s\t%d\t6\t60\t61\n" % r for r in refs))
    paths, lin = [], []
    for k in range(S):
        male = k % 2 == 0
        per_ref = []
        v = 100000
        for name, L in refs:
            nt = L // 16384 + 1
            if k == 3 and name == "2":
                nt -= 5                                            # a shorter sample: "0" columns
            scale = {"X": 0.5 if male else 1.0, "Y": 0.5 if male else 0.01}.get(name, 1.0)
            sizes = np.maximum(0, rng.normal(1.6e9 * scale, 1.5e8, nt)).astype(np.int64)
            iv = (v + np.concatenate([[0], np.cumsum(sizes)])).tolist()
            v = iv[-1]
            per_ref.append(iv if nt > 0 else [])
        p = tmp_path / ("smp%d.rest.bai" % k)
        p.write_bytes(make_bai(per_ref, [(1000 * (k + 1), 10 + k) for _ in refs]))
        paths.append(str(p)); lin.append(per_ref)
    return refs, str(fai), paths, lin


def oracle_depths(lin):
    """each sample's normalised depths per reference (I1-I3: sizes, capped weighted median, size / median)"""
    out = []
    for per_ref in lin:
        voff = np.array([v for r in per_ref for v in r], np.uint64)
        ptr = np.concatenate([[0], np.cumsum([len(r) for r in per_ref])]).astype(np.int64)
        sizes, sptr = orc.ic_sizes(voff, ptr)
        m = orc.ic_median(sizes)
        d = orc.ic_normalize(sizes, float(m))
        out.append([d[sptr[r]:sptr[r + 1]] for r in range(len(per_ref))])
    return out


def _xnorm(ds):
    S = len(ds)
    mat = np.zeros((S, max(len(d) for d in ds)), np.float32)
    for k in range(S):
        mat[k, :len(ds[k])] = ds[k]
    mat = orc.ic_xnorm(mat, np.array([len(d) for d in ds], np.int32))
    return [mat[k, :len(ds[k])] for k in range(S)]


def expected_outputs(refs, depths, names, order, extranorm):
    """(bed.gz lines, .roc text, bins S x 4) for the references in `order` (a reference may repeat, as `-c` makes it);
    NC* references are left out as the default --excludepatt does"""
    S = len(depths)
    rows = ["#chrom\tstart\tend\t" + "\t".join(names)]
    bins = np.zeros((S, 4), np.int64)
    roc_txt = ""
    for r in order:
        name, L = refs[r]
        if name.startswith("NC"):
            continue
        ds = [depths[k][r] for k in range(S)]
        longest = max(len(d) for d in ds)
        is_sex = name in ("X", "Y")
        if extranorm and not is_sex:
            ds = _xnorm(ds)
        for i in range(longest):
            rows.append("%s\t%d\t%d\t" % (name, i * 16384, (i + 1) * 16384) +
                        "\t".join("0" if i >= len(ds[k]) else "%.3g" % ds[k][i] for k in range(S)))
        if not is_sex:
            for k in range(S):
                bins[k] += orc.ic_bins(ds[k], longest)
        rocs = [orc.ic_roc(orc.ic_counts(ds[k])) for k in range(S)]
        roc_txt += "#chrom\tcov\t" + "\t".join(names) + "\n"
        for i in range(70):
            roc_txt += "%s\t%.2f\t" % (name, i / (70 * (2.0 / 3.0))) + "\t".join("%.2f" % rocs[k][i] for k in range(S)) + "\n"
    return rows, roc_txt, bins


def read_ped(out):
    stem = os.path.basename(str(out))
    return [ln.split("\t") for ln in open(os.path.join(str(out), stem + "-indexcov.ped")).read().splitlines()]


def check_ped_columns(ped, refs, depths, bins):
    """the header, the sex / CNX columns from X, the bins columns and the mapped / unmapped counts cohort_bais wrote"""
    S = len(depths)
    x = [n for n, _ in refs].index("X")
    assert ped[0][:8] == ["#family_id", "sample_id", "paternal_id", "maternal_id", "sex", "phenotype", "CNX", "CNY"]
    assert len(ped) == S + 1
    assert len({len(r) for r in ped}) == 1                        # num_colcounts == 1 (functional-tests.sh:26-30,50)
    col = ped[0].index("bins.out")
    for k in range(S):
        assert [int(v) for v in ped[k + 1][col:col + 4]] == bins[k].tolist(), k
        assert ped[k + 1][ped[0].index("CNX")] == "%.2f" % orc.ic_getcn(depths[k][x]), k
        assert ped[k + 1][4] == str(int(0.5 + orc.ic_getcn(depths[k][x]))), k
        assert ped[k + 1][-2:] == [str(1000 * (k + 1) * len(refs)), str((10 + k) * len(refs))], k


def expected_pcs(depths, names, extranorm, autosomes):
    """the oracle's (proj, sv, k) of the .ped PC columns: the byte matrix of the kept autosomes (after -n), then the SVD"""
    S = len(depths)
    refs = []
    for r, name in enumerate(names):
        if name not in autosomes:
            continue
        ds = [depths[k][r] for k in range(S)]
        refs.append(_xnorm(ds) if extranorm else ds)
    return op.pca(op.pca8_matrix(refs))


def compare_pcs(ped, proj, kk):
    """the PC1..PCk columns equal "%.2f" of the oracle's projections, except cells within 1e-7 of the column's largest
    magnitude from a half-cent boundary, which may be no more than twice what a uniform spread predicts (plus one)"""
    hdr = ped[0]
    c0 = hdr.index("p.out") + 1
    assert hdr[c0:c0 + kk] == ["PC%d" % (j + 1) for j in range(kk)]
    assert hdr[c0 + kk:] == ["mapped", "unmapped"]
    for j in range(kk):
        tol = 1e-7 * max(np.abs(proj[:, j]).max(), 1e-300)
        nr = op.half_cent_near(proj[:, j], tol)
        for k in range(len(ped) - 1):
            if not nr[k]:
                assert ped[k + 1][c0 + j] == "%.2f" % proj[k, j], (k, j, ped[k + 1][c0 + j], proj[k, j])
        assert nr.sum() <= 2 * len(nr) * min(1.0, 200 * tol) + 1
