#!/usr/bin/env bash
# make_reference_goldens.sh — on ANY box with `go` (>= 1.12) and `samtools` (>= 1.13) on PATH, build the unmodified
# reference (brentp/goleft v0.2.6) and write the outputs that pin this repo's oracle to the real thing:
#
#   tests/golden/ref_t_<W>.{depth,callable}.bed          goleft depth  -w W        on depth/test/t.bam   (.fai mode)
#   tests/golden/ref_t_bed_<W>.{depth,callable}.bed      goleft depth  -w W --bed  on depth/test/t.bam   (BED mode, windows.bed)
#   tests/golden/ref_hla_<W>.{depth,callable}.bed        goleft depth  -w W        on depth/test/hla.bam
#   tests/golden/ref_empty_<W>.{depth,callable}.bed      goleft depth  -w W        on a BAM without reads on the contig
#   tests/golden/ref_indexcov_sample27.{bed,roc,ped}     goleft indexcov           on indexcov/test-data/sample_issue_27.bam(.bai)
#   tests/golden/ref_depthwed.tsv                        goleft depthwed -s 1000   on two of the depth.bed files above
#   tests/golden/ref_multidepth_t_<chrom>.txt            multidepth -Q 1 --minsamples 0 -c chrom on t.bam (contigs with reads)
#   tests/golden/ref_dcnv_{depthwed,ties}.bed            dcnv on ref_depthwed.tsv and on dcnv_ties.tsv, with hg19.fa(.fai)
#   tests/golden/ref_emdepth_pow.txt                     the bits of math.Pow(i/2, 1.1), i = 1, 3..8, as Go computes them
#   tests/golden/ref_emdepth.{cn,cnv}.bed                our driver over the reference's emdepth package on emdepth_cohort.tsv
#                                                        (9 samples with planted CN1 / CN3 runs; ref_depthwed.tsv has 2 samples,
#                                                        where the reference's median32 panics)
#   tests/golden/ref_emdepth_gotest.txt                  `go test ./emdepth` (its TestBig fails: it expects CN 8, the code gives 9)
#   tests/golden/ref_indexcov_pca{8,4}.ped               goleft indexcov --fai on the .bai cohorts of tests/golden/make_pca_cohort.py
#   tests/golden/ref_cnveval_<case>_<mode>.txt           cnveval stdout on the sets of tests/golden/make_cnveval_sets.py
#   tests/golden/ref_csi_<bam>.bam.{bai,csi}, ref_csi_<bam>.m12.bam.csi
#                                                        samtools index -b / -c / -c -m 12 of depth/test/t.bam and hla.bam
#
# This image has neither toolchain (`go version`, `samtools --version`: command not found), so the files cannot be made
# here; until they exist every report says "bit-exact vs the restated oracle, parity unpinned".  tests/test_reference_goldens.py
# compares BOTH the oracle and the GPU output with these files when they are present and skips, loudly, when they are not.
#
#   usage: tools/make_reference_goldens.sh /path/to/goleft-checkout [outdir]
set -euo pipefail
REF=${1:?path to a brentp/goleft checkout (v0.2.6)}
OUT=${2:-$(cd "$(dirname "$0")/.." && pwd)/tests/golden}
command -v go >/dev/null || { echo "go not found" >&2; exit 2; }
command -v samtools >/dev/null || { echo "samtools not found" >&2; exit 2; }
ver=$(samtools --version | head -1 | awk '{print $2}')
case "$ver" in 0.*|1.[0-9]|1.[0-9].*|1.1[0-2]|1.1[0-2].*) echo "samtools $ver < 1.13: it caps depth at -d and prints zero-depth lines (SURVEY.md 8a D0); use >= 1.13" >&2; exit 2;; esac
mkdir -p "$OUT"
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
( cd "$REF" && CGO_ENABLED=0 go build -o "$TMP/goleft" ./cmd/goleft )
G="$TMP/goleft"
T="$REF/depth/test"

# reference FASTA index: goleft depth only reads <ref>.fai (depth.go:125-128); write one from the BAM header
fai_of() { samtools view -H "$1" | awk -F'\t' '$1=="@SQ"{n="";l=0;for(i=2;i<=NF;i++){if($i~/^SN:/)n=substr($i,4);if($i~/^LN:/)l=substr($i,4)}print n"\t"l"\t0\t60\t61"}' > "$2.fai"; }

# the reference's own tests run against test/hg19.fa(.fai) (depth/functional-test.sh:45); fall back to a .fai made from the header
if [[ -e "$T/hg19.fa.fai" ]]; then cp "$T/hg19.fa.fai" "$TMP/t.fa.fai"; else fai_of "$T/t.bam" "$TMP/t.fa"; fi
for W in 100 1000000000 55 60 71 13 2001 250; do      # depth/functional-test.sh:45-70 (+ the default 250)
  "$G" depth -Q 1 --ordered --windowsize $W --prefix "$TMP/t_$W" -r "$TMP/t.fa" "$T/t.bam"
  cp "$TMP/t_$W.depth.bed" "$OUT/ref_t_$W.depth.bed"; cp "$TMP/t_$W.callable.bed" "$OUT/ref_t_$W.callable.bed"
done
if [[ -e "$T/windows.bed" ]]; then
  for W in 10 1000000 50 55 60 71 13 2002; do         # depth/functional-test.sh:73-97
    "$G" depth -Q 1 --ordered --windowsize $W --bed "$T/windows.bed" --prefix "$TMP/tb_$W" -r "$TMP/t.fa" "$T/t.bam"
    cp "$TMP/tb_$W.depth.bed" "$OUT/ref_t_bed_$W.depth.bed"; cp "$TMP/tb_$W.callable.bed" "$OUT/ref_t_bed_$W.callable.bed"
  done
fi
if [[ -e "$T/hla.bam" ]]; then
  fai_of "$T/hla.bam" "$TMP/hla.fa"
  for W in 250 1000; do
    "$G" depth -Q 1 --ordered --windowsize $W --prefix "$TMP/hla_$W" -r "$TMP/hla.fa" "$T/hla.bam"
    cp "$TMP/hla_$W.depth.bed" "$OUT/ref_hla_$W.depth.bed"; cp "$TMP/hla_$W.callable.bed" "$OUT/ref_hla_$W.callable.bed"
  done
fi
# a contig without a single read: .fai lists one the BAM does not cover
printf 'nothing_here\t12345\t0\t60\t61\n' >> "$TMP/t.fa.fai"
"$G" depth -Q 1 --ordered -c nothing_here --windowsize 500 --prefix "$TMP/empty_500" -r "$TMP/t.fa" "$T/t.bam" || true
for f in depth callable; do [[ -e "$TMP/empty_500.nothing_here.$f.bed" ]] && cp "$TMP/empty_500.nothing_here.$f.bed" "$OUT/ref_empty_500.$f.bed"; done

cp "$TMP/t.fa.fai" "$OUT/ref_t.fai"
# samtools-written indexes of the same BAMs, a BAI and CSIs at min_shift 14 and 12, for tests/test_csi_goldens.py: the
# library's CSI reader against the BAI of one file (every CSI the other tests read comes from tests/csi_bams.py)
for B in "$T/t.bam" "$T/hla.bam"; do
  [[ -e "$B" ]] || continue
  n=$(basename "$B" .bam)
  cp "$B" "$TMP/$n.bam"
  samtools index -b "$TMP/$n.bam" "$OUT/ref_csi_$n.bam.bai"
  samtools index -c "$TMP/$n.bam" "$OUT/ref_csi_$n.bam.csi"
  samtools index -c -m 12 "$TMP/$n.bam" "$OUT/ref_csi_$n.m12.bam.csi"
done
IC="$REF/indexcov/test-data"
if [[ -e "$IC/sample_issue_27_0001.bam" ]]; then
  "$G" indexcov -d "$TMP/ic27" "$IC/sample_issue_27_0001.bam"
  zcat "$TMP/ic27/ic27-indexcov.bed.gz" > "$OUT/ref_indexcov_sample27.bed"
  cp "$TMP/ic27/ic27-indexcov.roc" "$OUT/ref_indexcov_sample27.roc"
  cut -f1-6,10- "$TMP/ic27/ic27-indexcov.ped" > "$OUT/ref_indexcov_sample27.ped" || cp "$TMP/ic27/ic27-indexcov.ped" "$OUT/ref_indexcov_sample27.ped"
fi
"$G" depthwed -s 1000 "$OUT/ref_t_100.depth.bed" "$OUT/ref_t_55.depth.bed" > "$OUT/ref_depthwed.tsv" || true
# multidepth is a separate binary of the reference (multidepth/multidepth.go); -Q 1 matches the committed decoded fixture
( cd "$REF" && CGO_ENABLED=0 go build -o "$TMP/multidepth" ./multidepth )
samtools idxstats "$T/t.bam" | awk -F'\t' '$3 > 0 {print $1}' | while read -r c; do
  "$TMP/multidepth" -Q 1 -p 1 --minsamples 0 -c "$c" "$T/t.bam" > "$OUT/ref_multidepth_t_$c.txt"
done
# dcnv is another separate binary (dcnv/dcnv.go); it writes depth.bed in its working directory.  hg19.fa(.fai) is the
# reference's own test FASTA, copied as a data fixture.  dcnv_ties.tsv: rows of 40 bases on chrM / chr22 share a few hundred
# GC values, so the order pdqsort leaves inside ties is pinned.
( cd "$REF" && CGO_ENABLED=0 go build -o "$TMP/dcnv" ./dcnv )
if [[ -e "$T/hg19.fa" && -e "$T/hg19.fa.fai" ]]; then
  cp "$T/hg19.fa" "$T/hg19.fa.fai" "$OUT/"
  awk -F'\t' 'BEGIN{OFS="\t"; srand(7); printf "#chrom\tstart\tend"; for(i=0;i<7;i++) printf "\ts%d", i; print ""}
       $1=="chrM" || $1=="chr22" {n=0; for(a=0; a+40<$2 && n<2000; a+=40){n++; printf "%s\t%d\t%d", $1, a, a+40; for(i=0;i<7;i++) printf "\t%d", int(rand()*60); print ""}}' \
      "$T/hg19.fa.fai" > "$OUT/dcnv_ties.tsv"
  for c in depthwed:ref_depthwed.tsv ties:dcnv_ties.tsv; do
    ( cd "$TMP" && "$TMP/dcnv" "$OUT/${c#*:}" "$OUT/hg19.fa" >/dev/null && cp depth.bed "$OUT/ref_dcnv_${c%%:*}.bed" ) || true
  done
fi
# emdepth is a library of the reference with no command.  The driver below (ours, DESIGN §1.10) builds against a copy of
# the package's non-test sources made here at run time: one Cache over the rows in file order, Clear(nil) at every
# chromosome change and at the end, the CNVs of one Clear in sample order.  It writes P.cn.bed / P.cnv.bed as
# `goleft emdepth --prefix P` does, and prints the Pow bits.
mkdir -p "$TMP/emdrv/emdepth"
cp "$REF"/emdepth/emdepth.go "$REF"/emdepth/stats.go "$TMP/emdrv/emdepth/"
printf 'module emdrv\n\ngo 1.12\n' > "$TMP/emdrv/go.mod"
cat > "$TMP/emdrv/main.go" <<'GO'
package main

import (
	"bufio"
	"fmt"
	"math"
	"os"
	"sort"
	"strconv"
	"strings"

	"emdrv/emdepth"
)

type row struct {
	chrom      string
	start, end uint32
}

func main() {
	if os.Args[1] == "pow" {
		for _, i := range []int{1, 3, 4, 5, 6, 7, 8} {
			fmt.Printf("%x\n", math.Float64bits(math.Pow(float64(i)/2, 1.1)))
		}
		return
	}
	f, err := os.Open(os.Args[1])
	if err != nil {
		panic(err)
	}
	prefix := os.Args[2]
	cn, _ := os.Create(prefix + ".cn.bed")
	cnv, _ := os.Create(prefix + ".cnv.bed")
	wcn, wcnv := bufio.NewWriter(cn), bufio.NewWriter(cnv)
	fmt.Fprintln(wcnv, "#chrom\tstart\tend\tsample\tn\tcns\tpsize")
	br := bufio.NewReader(f)
	var samples []string
	var rows []row
	var cache emdepth.Cache
	emit := func(cs []*emdepth.CNV) {
		sort.Slice(cs, func(a, b int) bool { return cs[a].SampleI < cs[b].SampleI })
		for _, c := range cs {
			p0, p1 := c.Position[0], c.Position[len(c.Position)-1]
			chrom := ""
			for k := len(rows) - 1; k >= 0; k-- { // the most recent row at the first kept position
				if rows[k].start == p0.Start && rows[k].end == p0.End {
					chrom = rows[k].chrom
					break
				}
			}
			cns := make([]string, len(c.CN))
			for k, v := range c.CN {
				cns[k] = strconv.Itoa(v)
			}
			fmt.Fprintf(wcnv, "%s\t%d\t%d\t%s\t%d\t%s\t%d\n", chrom, p0.Start, p1.End, samples[c.SampleI], len(c.CN), strings.Join(cns, ","), c.PSize)
		}
	}
	for {
		line, err := br.ReadString('\n')
		if err != nil {
			break
		}
		if len(rows) == 0 && (line[0] == '#' || strings.HasPrefix(line, "chrom")) {
			h := strings.Split(strings.TrimSpace(line), "\t")
			samples = h[3:]
			fmt.Fprintln(wcn, strings.Join(h, "\t"))
			continue
		}
		toks := strings.Split(strings.TrimSpace(line), "\t")
		s, _ := strconv.Atoi(toks[1])
		e, _ := strconv.Atoi(toks[2])
		r := row{toks[0], uint32(s), uint32(e)}
		if len(rows) > 0 && rows[len(rows)-1].chrom != r.chrom {
			emit(cache.Clear(nil))
		}
		rows = append(rows, r)
		d := make([]float32, len(toks)-3)
		for k, t := range toks[3:] {
			v, err := strconv.ParseFloat(t, 64)
			if err != nil {
				panic(err)
			}
			d[k] = float32(v)
		}
		em := emdepth.EMDepth(d, emdepth.Position{Start: r.start, End: r.end})
		c := em.CN()
		out := make([]string, len(c))
		for k, v := range c {
			out[k] = strconv.Itoa(v)
		}
		fmt.Fprintf(wcn, "%s\t%d\t%d\t%s\n", r.chrom, r.start, r.end, strings.Join(out, "\t"))
		emit(cache.Add(em))
	}
	emit(cache.Clear(nil))
	wcn.Flush()
	wcnv.Flush()
	cn.Close()
	cnv.Close()
}
GO
( cd "$TMP/emdrv" && CGO_ENABLED=0 go build -o "$TMP/emdrv_bin" . )
"$TMP/emdrv_bin" pow > "$OUT/ref_emdepth_pow.txt"
awk 'BEGIN{OFS="\t"; srand(11); printf "#chrom\tstart\tend"; for(i=0;i<9;i++) printf "\ts%d", i; print ""
     for(c=1;c<=2;c++) for(r=0;r<(c==1?2000:1000);r++){printf "chr%d\t%d\t%d", c, r*1000, r*1000+1000
       for(i=0;i<9;i++){v=30+rand()*10; if(c==1&&i==3&&r>=500&&r<540) v/=2; if(c==2&&i==6&&r>=100&&r<130) v*=1.5; printf "\t%d", int(v)}
       print ""}}' > "$OUT/emdepth_cohort.tsv"
"$TMP/emdrv_bin" "$OUT/emdepth_cohort.tsv" "$TMP/em" && cp "$TMP/em.cn.bed" "$OUT/ref_emdepth.cn.bed" && cp "$TMP/em.cnv.bed" "$OUT/ref_emdepth.cnv.bed" || true
( cd "$REF" && go test ./emdepth 2>&1 || true ) > "$OUT/ref_emdepth_gotest.txt"
# indexcov's PC1..PC5 .ped columns (indexcov.go:773-807): the full .ped of two generated .bai cohorts with planted groups,
# 8 samples and 4 samples (rank 3 after centring: the reference's 4th column is a constant).  tests/golden/make_pca_cohort.py
# writes the same bytes wherever it runs; tests/test_reference_goldens_indexcov_pca.py regenerates them for our side.
python3 "$(dirname "$0")/../tests/golden/make_pca_cohort.py" "$TMP/pcac"
for c in pca8 pca4; do
  "$G" indexcov -d "$TMP/$c" --fai "$TMP/pcac/g.fa.fai" "$TMP/pcac/$c"/s*.bai && cp "$TMP/$c/$c-indexcov.ped" "$OUT/ref_indexcov_$c.ped" || true
done
# cnveval (cnveval/cmd/cnveval): stdout on the sets tests/golden/make_cnveval_sets.py writes, for each argument list of
# its MODES.  Run inside $TMP: the reference writes its CPU profile x.cpu.pprof into the working directory.
( cd "$REF" && CGO_ENABLED=0 go build -o "$TMP/cnveval" ./cnveval/cmd/cnveval )
python3 "$(dirname "$0")/../tests/golden/make_cnveval_sets.py" "$TMP/cnv"
for c in cohort quirks; do
  for m in default:"" limit:"-s" m05:"-m 0.5"; do
    # shellcheck disable=SC2086
    ( cd "$TMP" && "$TMP/cnveval" ${m#*:} "$TMP/cnv/$c.truth.bed" "$TMP/cnv/$c.test.bed" > "$OUT/ref_cnveval_${c}_${m%%:*}.txt" ) || rm -f "$OUT/ref_cnveval_${c}_${m%%:*}.txt"
  done
done
samtools --version | head -1 > "$OUT/ref_PROVENANCE.txt"; go version >> "$OUT/ref_PROVENANCE.txt"; (cd "$REF" && git rev-parse HEAD 2>/dev/null || true) >> "$OUT/ref_PROVENANCE.txt"
echo "wrote $(ls "$OUT"/ref_* | wc -l) files to $OUT"
