"""`goleft indexcov`'s PC1..PC5 .ped columns end to end (indexcov.go:686-705,773-807,842-890): the CLI on .bai and .crai
cohorts against the oracle's depths (oracle/loader.py), byte matrix and SVD route (oracle/indexcov_pca.py)."""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bamutil import make_bai  # noqa: E402
from indexcov_cli_oracle import compare_pcs, expected_pcs, oracle_depths, read_ped  # noqa: E402
from oracle import indexcov_pca as op  # noqa: E402
from oracle import loader as orc  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
REFS = [("1", 3_000_000), ("2", 2_000_000), ("GL000207.1", 4262), ("X", 1_500_000), ("Y", 600_000), ("NC_007605", 171823)]


def run(*args, env=None):
    p = subprocess.run([GOLEFT, *args], capture_output=True, text=True, env=dict(os.environ, **env) if env else None)
    assert p.returncode == 0, p.stderr
    return p


def _cohort(tmp_path, S, seed=1):
    """S samples in three groups: each group loses coverage over its own stretch of chromosome 1 (planted structure for
    the components); one sample is short on chromosome 2"""
    rng = np.random.default_rng(seed)
    fai = tmp_path / "g.fa.fai"
    fai.write_text("".join("%s\t%d\t6\t60\t61\n" % r for r in REFS))
    paths, lin = [], []
    for k in range(S):
        grp = k % 3
        per_ref = []
        v = 100000
        for name, L in REFS:
            nt = L // 16384 + 1
            if k == 1 and name == "2":
                nt -= 7
            scale = {"X": 0.5 if k % 2 == 0 else 1.0, "Y": 0.5 if k % 2 == 0 else 0.01}.get(name, 1.0)
            mean = np.full(nt, 1.6e9 * scale)
            if name == "1":
                mean[30 + 40 * grp:60 + 40 * grp] *= 0.35 + 0.1 * grp
            sizes = np.maximum(0, rng.normal(mean, 1.2e8)).astype(np.int64)
            iv = [v]
            for sz in sizes:
                v += int(sz); iv.append(v)
            per_ref.append(iv)
        p = tmp_path / ("smp%d.rest.bai" % k)
        p.write_bytes(make_bai(per_ref, [(1000 * (k + 1), 10 + k) for _ in REFS]))
        paths.append(str(p)); lin.append(per_ref)
    return str(fai), paths, lin


@pytest.mark.parametrize("extranorm", [False, True])
def test_ped_pcs_against_oracle(tmp_path, extranorm):
    fai, paths, lin = _cohort(tmp_path, 9)
    out = tmp_path / "pp"
    p = run("indexcov", "-d", str(out), "--fai", fai, *(["-n"] if extranorm else []), *paths)
    assert "principal components" not in p.stderr
    proj, sv, kk = expected_pcs(oracle_depths(lin), [n for n, _ in REFS], extranorm, {"1", "2", "GL000207.1"})
    assert kk == 5 and sv[4] > 0
    compare_pcs(read_ped(out), proj, kk)


@pytest.mark.parametrize("S", [1, 2, 3, 4])
def test_few_samples(tmp_path, S):
    fai, paths, lin = _cohort(tmp_path, S)
    out = tmp_path / "fs"
    p = run("indexcov", "-d", str(out), "--fai", fai, *paths)
    assert "got: %d principal components" % S in p.stderr
    ped = read_ped(out)
    if S < 3:
        assert "indexcov: %d principal components, not plotting" % S in p.stderr
        assert not any(h.startswith("PC") for h in ped[0])
        return
    assert "not plotting" not in p.stderr
    proj, sv, kk = expected_pcs(oracle_depths(lin), [n for n, _ in REFS], False, {"1", "2", "GL000207.1"})
    assert kk == S and sv[S - 1] == 0                                  # rank S - 1 after centring: the last column is 0.00
    compare_pcs(ped, proj, kk)
    c0 = ped[0].index("p.out") + 1
    assert all(r[c0 + S - 1] == "0.00" for r in ped[1:])


def test_no_autosome_kept(tmp_path):
    """--excludepatt removes every autosome: D = 0, no PC columns, exit 0 (the reference's gonum panics here)"""
    fai, paths, _ = _cohort(tmp_path, 5)
    out = tmp_path / "na"
    p = run("indexcov", "-d", str(out), "--fai", fai, "--excludepatt", "^(1|2|GL.*|NC.*)$", *paths)
    assert "got: 0 principal components" in p.stderr and "indexcov: 0 principal components, not plotting" in p.stderr
    assert not any(h.startswith("PC") for h in read_ped(out)[0])


def test_crai_cohort(tmp_path):
    rng = np.random.default_rng(9)
    refs = [("1", 4_000_000), ("2", 2_500_000)]
    fai = tmp_path / "g.fa.fai"
    fai.write_text("".join("%s\t%d\t6\t60\t61\n" % r for r in refs))
    paths, slices = [], []
    for k in range(6):
        per, lines = [], []
        for si, (name, L) in enumerate(refs):
            st = np.cumsum(rng.integers(150_000, 400_000, 9)).astype(np.int64) + 1
            st = st[st < L - 10]
            sp = rng.integers(200_000, 420_000, st.size).astype(np.int64)
            by = rng.integers(2_000_000, 4_000_000, st.size).astype(np.int32)
            per.append((st, sp, by))
            lines += ["%d\t%d\t%d\t%d\t%d\t%d\n" % (si, a, b, 1000 + i, 10, c) for i, (a, b, c) in enumerate(zip(st, sp, by))]
        p = tmp_path / ("cram%d.crai" % k)
        p.write_bytes(gzip.compress("".join(lines).encode()))
        paths.append(str(p)); slices.append(per)
    out = tmp_path / "cc"
    run("indexcov", "-d", str(out), "--fai", str(fai), *paths)
    depths = []
    for k in range(6):
        sz = [orc.crai_sizes(*slices[k][r]) for r in range(2)]
        m = orc.ic_median(np.concatenate(sz))
        depths.append([orc.ic_normalize(x, float(m)) for x in sz])
    proj, sv, kk = expected_pcs(depths, ["1", "2"], False, {"1", "2"})
    ped = read_ped(out)
    hdr = ped[0]
    c0 = hdr.index("p.out") + 1
    assert hdr[c0:] == ["PC%d" % (j + 1) for j in range(kk)]          # CRAM indexes carry no mapped / unmapped counts
    for j in range(kk):
        tol = 1e-7 * max(np.abs(proj[:, j]).max(), 1e-300)
        nr = op.half_cent_near(proj[:, j], tol)
        assert all(ped[k + 1][c0 + j] == "%.2f" % proj[k, j] for k in range(6) if not nr[k])


def test_gpus_same_bytes(tmp_path):
    fai, paths, _ = _cohort(tmp_path, 11, seed=5)
    outs = []
    for g in (1, 3):
        out = tmp_path / ("g%d" % g) / "tt"
        os.makedirs(str(out.parent))
        run("indexcov", "-d", str(out), "--gpus", str(g), "--fai", fai, *paths, env={"GL_OVERSUBSCRIBE": "1"})
        outs.append(open(str(out / "tt-indexcov.ped"), "rb").read())
    assert outs[0] == outs[1] and b"PC5" in outs[0]
