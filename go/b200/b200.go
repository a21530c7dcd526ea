// Package b200 binds libgoleft_b200.so (CUDA, sm_90a) for goleft's windowed-depth path.
//
// SOURCE ONLY: the build image of this repository has no Go toolchain (`go: command not found`), so this file has never
// been compiled there; the same C ABI (include/goleft_b200.h) is exercised by the C++ CLI (cli/goleft.cpp) and by the
// ctypes binding the tests use (goleft_b200/capi.py).  Build with CGO_ENABLED=1 after `make lib`.
//
// What the reference would call (paths in brentp/goleft v0.2.6):
//   depth/depth.go:392-394  process.Runner(genCommands(args), ...) + callback :238-364
//        -> Bam.DepthContig per reference sequence (decode + count + window means + callable runs + BED text on the GPU)
//   indexcov/indexcov.go:417-434,651-676  Index.init / NormalizedDepth / CountsAtDepth
//        -> Ctx.IndexcovCohort (+ gl_indexcov_counts_batch, gl_indexcov_xnorm, gl_format_g3)
package b200

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../goleft_b200 -lgoleft_b200 -Wl,-rpath,${SRCDIR}/../../goleft_b200
#include <stdlib.h>
#include "goleft_b200.h"
*/
import "C"

import (
	"fmt"
	"runtime"
	"unsafe"
)

// Ctx is one GPU context; not safe for concurrent use (one goroutine at a time, like gl_ctx).
type Ctx struct{ h *C.gl_ctx }

// DeviceCount is the number of visible CUDA devices (goleft depth deals contigs to all of them).
func DeviceCount() int {
	var n C.int
	if C.gl_device_count(&n) != C.GL_OK {
		return 0
	}
	return int(n)
}

// New creates a context on one GPU.  There is no CPU fallback: without a device this fails.
func New(device int) (*Ctx, error) {
	var h *C.gl_ctx
	if rc := C.gl_ctx_create(C.int(device), &h); rc != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: %s", C.GoString(C.gl_last_error(nil)))
	}
	c := &Ctx{h}
	runtime.SetFinalizer(c, func(c *Ctx) { C.gl_ctx_destroy(c.h) })
	return c, nil
}

func (c *Ctx) err(rc C.int) error {
	if rc == C.GL_OK {
		return nil
	}
	return fmt.Errorf("goleft_b200: %s", C.GoString(C.gl_last_error(c.h)))
}

// LptAssign deals work items (contigs, weight = length) to `bins` GPUs, longest first onto the least loaded one.
func LptAssign(weights []int64, bins int) []int32 {
	out := make([]int32, len(weights))
	if len(weights) == 0 {
		return out
	}
	C.gl_lpt_assign((*C.int64_t)(unsafe.Pointer(&weights[0])), C.int32_t(len(weights)), C.int32_t(bins),
		(*C.int32_t)(unsafe.Pointer(&out[0])), nil)
	return out
}

// Bam is an indexed BAM opened by the library's feeder (BGZF inflate + record parse on the host pool).
type Bam struct{ h *C.gl_bam }

// OpenBam opens path and its .bai.  The index is what `samtools depth -r` needs too (depth/depth.go:116,152).
func OpenBam(path string) (*Bam, error) {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	var h *C.gl_bam
	buf := make([]byte, 512)
	if rc := C.gl_bam_open(cs, &h, (*C.char)(unsafe.Pointer(&buf[0])), 512); rc != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: %s", C.GoString((*C.char)(unsafe.Pointer(&buf[0]))))
	}
	b := &Bam{h}
	runtime.SetFinalizer(b, func(b *Bam) { C.gl_bam_close(b.h) })
	return b, nil
}

// DepthContig replaces, for one reference sequence, every `samtools depth -Q q -r chrom:b-e` child of
// depth/depth.go:129-159 and the callback of :238-364 run on each of its chunks: it returns the bytes the reference
// appends to <prefix>.depth.bed and <prefix>.callable.bed for that sequence (chunks of `step` bases, depth.go:132).
func (c *Ctx) DepthContig(b *Bam, tid int, chrom string, length int, window, minCov, maxMeanDepth, q int) (depthBed, callableBed []byte, err error) {
	step := 10000000 / window * window
	if step < window {
		step = window
	}
	cs := C.CString(chrom)
	defer C.free(unsafe.Pointer(cs))
	nWin := (length-1)/window + 1
	depthBed = make([]byte, int(C.gl_depth_text_bound(cs, C.int64_t(nWin))))
	callableBed = make([]byte, 1<<20)
	var seg C.gl_bam_segments
	// The feeder on the GPU first (BGZF inflate + record parse + filter + CIGAR walk on the device: only compressed bytes
	// cross PCIe); GL_ESTATE means this reference cannot take that road (no usable index, a member the device inflater
	// rejects) and the host feeder below decodes it.
	var dS, dE *C.int32_t
	var dN C.int64_t
	if rc := C.gl_bam_decode_device(c.h, b.h, C.int32_t(tid), C.int32_t(q), &dS, &dE, &dN, &seg); rc == C.GL_OK {
		if e := c.err(C.gl_depth_begin(c.h, 0, C.int64_t(length))); e != nil {
			return nil, nil, e
		}
		if dN > 0 {
			if e := c.err(C.gl_depth_add_segments_device(c.h, dS, dE, dN)); e != nil {
				return nil, nil, e
			}
		}
		if e := c.err(C.gl_depth_reduce(c.h, C.int32_t(window), C.int32_t(minCov), C.int32_t(maxMeanDepth), C.int64_t(step))); e != nil {
			return nil, nil, e
		}
		for attempt := 0; attempt < 2; attempt++ {
			var dl, cl C.int64_t
			rc := C.gl_depth_text(c.h, cs, (*C.char)(unsafe.Pointer(&depthBed[0])), C.int64_t(len(depthBed)), &dl,
				(*C.char)(unsafe.Pointer(&callableBed[0])), C.int64_t(len(callableBed)), &cl)
			if rc == C.GL_ERANGE && attempt == 0 {
				depthBed = make([]byte, int(dl)+16)
				callableBed = make([]byte, int(cl)+16)
				continue
			}
			if e := c.err(rc); e != nil {
				return nil, nil, e
			}
			return depthBed[:dl], callableBed[:cl], nil
		}
	} else if rc != C.GL_ESTATE {
		return nil, nil, c.err(rc)
	}
	ebuf := make([]byte, 512)
	if rc := C.gl_bam_decode(b.h, C.int32_t(tid), 0, C.int64_t(length), C.int32_t(q), 0, 0, &seg, (*C.char)(unsafe.Pointer(&ebuf[0])), 512); rc != C.GL_OK {
		return nil, nil, fmt.Errorf("goleft_b200: %s", C.GoString((*C.char)(unsafe.Pointer(&ebuf[0]))))
	}
	for attempt := 0; attempt < 2; attempt++ {
		var dl, cl C.int64_t
		var rc C.int
		dp := (*C.char)(unsafe.Pointer(&depthBed[0]))
		cp := (*C.char)(unsafe.Pointer(&callableBed[0]))
		if seg.format == 8 {
			rc = C.gl_depth_bed_contig_packed8(c.h, cs, C.int64_t(length), seg.a0, (*C.uint8_t)(seg.a1), (*C.uint8_t)(seg.a2), seg.n,
				C.int32_t(window), C.int32_t(minCov), C.int32_t(maxMeanDepth), C.int64_t(step),
				dp, C.int64_t(len(depthBed)), &dl, cp, C.int64_t(len(callableBed)), &cl)
		} else {
			rc = C.gl_depth_bed_contig(c.h, cs, C.int64_t(length), seg.a0, (*C.int32_t)(seg.a1), seg.n,
				C.int32_t(window), C.int32_t(minCov), C.int32_t(maxMeanDepth), C.int64_t(step), 0,
				dp, C.int64_t(len(depthBed)), &dl, cp, C.int64_t(len(callableBed)), &cl)
		}
		if rc == C.GL_ERANGE && attempt == 0 {
			depthBed = make([]byte, int(dl)+16)
			callableBed = make([]byte, int(cl)+16)
			continue
		}
		if e := c.err(rc); e != nil {
			return nil, nil, e
		}
		return depthBed[:dl], callableBed[:cl], nil
	}
	return nil, nil, fmt.Errorf("goleft_b200: text buffers did not converge")
}

// DepthRegion replaces one `samtools depth -r chrom:rs+1-re` child plus the per-line loop of the callback
// (depth/depth.go:45,238-364): window sums and class runs for [rs,re).  start/end are the M/=/X blocks of
// the records that pass the flag/MAPQ filter (what biogo's bam.Reader + Cigar walk yields).
func (c *Ctx) DepthRegion(rs, re int, start, end []int32, window, minCov, maxMeanDepth, runBreak int) (sums []int64, runStart []int32, runClass []uint8, err error) {
	nWin := (re-1)/window - rs/window + 1
	sums = make([]int64, nWin)
	cap := 1 << 16
	for {
		runStart = make([]int32, cap)
		runClass = make([]uint8, cap)
		var nw, nr C.int64_t
		var ps, pe *C.int32_t
		if len(start) > 0 {
			ps = (*C.int32_t)(unsafe.Pointer(&start[0]))
			pe = (*C.int32_t)(unsafe.Pointer(&end[0]))
		}
		rc := C.gl_depth_region(c.h, C.int64_t(rs), C.int64_t(re), ps, pe, C.int64_t(len(start)),
			C.int32_t(window), C.int32_t(minCov), C.int32_t(maxMeanDepth), C.int64_t(runBreak),
			(*C.int64_t)(unsafe.Pointer(&sums[0])), C.int64_t(nWin), &nw,
			(*C.int32_t)(unsafe.Pointer(&runStart[0])), (*C.uint8_t)(unsafe.Pointer(&runClass[0])), C.int64_t(cap), &nr)
		if rc == C.GL_ERANGE && int(nr) > cap {
			cap = int(nr) + 1024
			continue
		}
		if e := c.err(rc); e != nil {
			return nil, nil, nil, e
		}
		return sums[:nw], runStart[:nr], runClass[:nr], nil
	}
}

// FormatChunk returns exactly the rows the reference's callback writes for one chunk (depth.go:293-358), BED-mode
// chunk-edge quirks included (host-side; DepthContig formats on the GPU).
func FormatChunk(chrom string, rs, re, window int, sums []int64, runStart []int32, runClass []uint8) (depthBed, callableBed string) {
	cs := C.CString(chrom)
	defer C.free(unsafe.Pointer(cs))
	var d, ca *C.char
	var dl, cl C.int64_t
	C.gl_depth_format_chunk(cs, C.int64_t(rs), C.int64_t(re), C.int32_t(window),
		(*C.int64_t)(unsafe.Pointer(&sums[0])), C.int64_t(len(sums)),
		(*C.int32_t)(unsafe.Pointer(&runStart[0])), (*C.uint8_t)(unsafe.Pointer(&runClass[0])), C.int64_t(len(runStart)),
		&d, &dl, &ca, &cl)
	defer C.gl_free_text(d)
	defer C.gl_free_text(ca)
	return C.GoStringN(d, C.int(dl)), C.GoStringN(ca, C.int(cl))
}

// IndexcovCohort replaces Index.init + NormalizedDepth for every sample at once
// (indexcov/indexcov.go:83-151): sizes in CSR layout by sample.
func (c *Ctx) IndexcovCohort(sizes []int64, samplePtr []int64) (medians []float64, depths []float32, err error) {
	S := len(samplePtr) - 1
	medians = make([]float64, S)
	depths = make([]float32, len(sizes))
	rc := C.gl_indexcov_cohort(c.h, (*C.int64_t)(unsafe.Pointer(&sizes[0])), (*C.int64_t)(unsafe.Pointer(&samplePtr[0])),
		C.int32_t(S), (*C.double)(unsafe.Pointer(&medians[0])), (*C.float)(unsafe.Pointer(&depths[0])))
	return medians, depths, c.err(rc)
}

// Multidepth replaces multidepth/multidepth.go:208-283 for one contig of `length` bases: addSegments(i) must add sample i's
// M/=/X blocks (records with Flags&0x704 == 0 && MapQ >= Q) to the open region with gl_depth_add_segments* — it is called
// twice per sample, once per pass.  Returns the rows after the header line, exactly as the reference with -p 1.
func (c *Ctx) Multidepth(chrom string, length, samples, minCov int, minSamples float64, maxSkip, minSize, window int,
	addSegments func(i int) error) ([]byte, error) {
	if err := c.err(C.gl_multidepth_begin(c.h, C.int64_t(length), C.int32_t(samples), C.int32_t(minCov), C.double(minSamples))); err != nil {
		return nil, err
	}
	pass := func(f func(i int) C.int) error {
		for i := 0; i < samples; i++ {
			if err := c.err(C.gl_depth_begin(c.h, 0, C.int64_t(length))); err != nil {
				return err
			}
			if err := addSegments(i); err != nil {
				return err
			}
			if err := c.err(f(i)); err != nil {
				return err
			}
		}
		return nil
	}
	if err := pass(func(int) C.int { return C.gl_multidepth_count(c.h) }); err != nil {
		return nil, err
	}
	var nr C.int64_t
	if err := c.err(C.gl_multidepth_sites(c.h, nil, nil, 0, &nr)); err != nil {
		return nil, err
	}
	rs, rc := make([]int32, nr+1), make([]uint8, nr+1)
	if err := c.err(C.gl_multidepth_sites(c.h, (*C.int32_t)(&rs[0]), (*C.uint8_t)(&rc[0]), nr, &nr)); err != nil {
		return nil, err
	}
	var nb C.int64_t
	if C.gl_multidepth_blocks((*C.int32_t)(&rs[0]), (*C.uint8_t)(&rc[0]), nr, C.int64_t(length), C.int32_t(samples), 0, C.int64_t(maxSkip),
		C.int64_t(minSize), C.int64_t(window), nil, nil, nil, 0, &nb) != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: gl_multidepth_blocks failed")
	}
	bs, be, bn := make([]int64, nb+1), make([]int64, nb+1), make([]int64, nb+1)
	C.gl_multidepth_blocks((*C.int32_t)(&rs[0]), (*C.uint8_t)(&rc[0]), nr, C.int64_t(length), C.int32_t(samples), 0, C.int64_t(maxSkip),
		C.int64_t(minSize), C.int64_t(window), (*C.int64_t)(&bs[0]), (*C.int64_t)(&be[0]), (*C.int64_t)(&bn[0]), nb, &nb)
	if err := c.err(C.gl_multidepth_set_blocks(c.h, (*C.int64_t)(&bs[0]), (*C.int64_t)(&be[0]), (*C.int64_t)(&bn[0]), nb)); err != nil {
		return nil, err
	}
	if err := pass(func(i int) C.int { return C.gl_multidepth_sums(c.h, C.int32_t(i)) }); err != nil {
		return nil, err
	}
	cells := int(nb)*samples + 1
	q, val, cert := make([]int64, cells), make([]float64, cells), make([]uint8, cells)
	if err := c.err(C.gl_multidepth_result(c.h, nil, (*C.int64_t)(&q[0]), (*C.double)(&val[0]), (*C.uint8_t)(&cert[0]))); err != nil {
		return nil, err
	}
	cs := C.CString(chrom)
	defer C.free(unsafe.Pointer(cs))
	var text *C.char
	var tl C.int64_t
	if C.gl_multidepth_text(cs, (*C.int64_t)(&bs[0]), (*C.int64_t)(&be[0]), nb, C.int32_t(samples), (*C.int64_t)(&q[0]), (*C.double)(&val[0]),
		(*C.uint8_t)(&cert[0]), 0, &text, &tl) != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: gl_multidepth_text failed")
	}
	defer C.gl_free_text(text)
	return C.GoBytes(unsafe.Pointer(text), C.int(tl)), nil
}

// MultidepthMerge adds the pass-1 counters, site bits and counted samples of every src context into c's, for a multidepth
// run whose samples were counted on several contexts (any devices) begun with the same parameters.  Each src then refuses
// counts, sites and merges until it adopts c's sites with MultidepthAdoptSites.
func (c *Ctx) MultidepthMerge(src []*Ctx) error {
	if len(src) == 0 {
		return c.err(C.gl_multidepth_merge(c.h, nil, 0))
	}
	hs := make([]*C.gl_ctx, len(src))
	for i, s := range src {
		hs[i] = s.h
	}
	return c.err(C.gl_multidepth_merge(c.h, (**C.gl_ctx)(unsafe.Pointer(&hs[0])), C.int32_t(len(src))))
}

// MultidepthAdoptSites copies src's site and sufficient bits and class runs into c; src must have run its sites.  c then
// takes the blocks and sums its own samples (with their cohort numbers) as if it had run its sites itself.
func (c *Ctx) MultidepthAdoptSites(src *Ctx) error {
	return c.err(C.gl_multidepth_adopt_sites(c.h, src.h))
}

// Dcnv replaces GeneralDebiaser.Sort / Debias / Unsort + NormalizeBySampleMedian of dcnv/dcnv.go:329-337 on the
// n x S row-major depth matrix `depths` (rows in position order; normalised in place), with gcs the GC fraction of each row.
// The argsort is Go's own sort.Sort order (gl_go_argsort_f64), so floats.Argsort may equally be used.  Returns the sample
// medians; fmt.Sprintf("%.2f") of the result is what dcnv writes, or FormatF2 gives the same text as 16-byte tokens.
func (c *Ctx) Dcnv(depths []float64, gcs []float64, samples int) ([]float64, error) {
	n := len(gcs)
	inds := make([]int64, n)
	if C.gl_go_argsort_f64((*C.double)(&gcs[0]), C.int64_t(n), (*C.int64_t)(&inds[0])) != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: gl_go_argsort_f64 failed")
	}
	medians := make([]float64, samples)
	d := (*C.double)(unsafe.Pointer(&depths[0]))
	rc := C.gl_dcnv_normalize(c.h, d, C.int64_t(n), C.int64_t(samples), (*C.int64_t)(&inds[0]), 0, C.int32_t(samples), 0, d,
		C.int64_t(samples), (*C.double)(&medians[0]))
	return medians, c.err(rc)
}

// DcnvChunk is Dcnv with ChunkDebiaser.Debias (dcnv/debiaser/debiaser.go:125-170, ScoreWindow = window) in place of the
// moving median, over the rows in GC order (`goleft dcnv --chunk W`): the sorted rows are cut into chunks spanning at most
// window of GC, and each sample's values in a chunk are divided by their median there when it is > 0.  window must be
// finite and > 0.  Returns the sample medians of the later NormalizeBySampleMedian.
func (c *Ctx) DcnvChunk(depths []float64, gcs []float64, samples int, window float64) ([]float64, error) {
	n := len(gcs)
	inds := make([]int64, n)
	if C.gl_go_argsort_f64((*C.double)(&gcs[0]), C.int64_t(n), (*C.int64_t)(&inds[0])) != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: gl_go_argsort_f64 failed")
	}
	sorted := make([]float64, n)
	for i, j := range inds {
		sorted[i] = gcs[j]
	}
	var nChunks C.int64_t
	if C.gl_dcnv_chunk_slices((*C.double)(&sorted[0]), C.int64_t(n), C.double(window), nil, 0, &nChunks) != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: gl_dcnv_chunk_slices: window must be finite and > 0")
	}
	ptr := make([]int64, int(nChunks)+1)
	if C.gl_dcnv_chunk_slices((*C.double)(&sorted[0]), C.int64_t(n), C.double(window), (*C.int64_t)(&ptr[0]), C.int64_t(len(ptr)),
		&nChunks) != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: gl_dcnv_chunk_slices failed")
	}
	medians := make([]float64, samples)
	d := (*C.double)(unsafe.Pointer(&depths[0]))
	rc := C.gl_dcnv_normalize_chunked(c.h, d, C.int64_t(n), C.int64_t(samples), (*C.int64_t)(&inds[0]), (*C.int64_t)(&ptr[0]), nChunks,
		0, C.int32_t(samples), 0, d, C.int64_t(samples), (*C.double)(&medians[0]))
	return medians, c.err(rc)
}

// DcnvSVD replaces scalers.ZScore.Scale + debiaser.SVD{MinVariancePct}.Debias + ZScore.UnScale (dcnv/scalers/scalers.go:25-56,
// dcnv/debiaser/debiaser.go:173-200) on the normalised n x S row-major matrix `depths`, in place: rows whose values are all
// equal are left as they are, the leading components whose share of the singular values is above minPct (at most 15) are
// removed from the z-scores of the others.  Returns the S singular values and how many components were removed; the
// reference logs "variance:" with 100 s[i] / sum(s) of each removed one.
func (c *Ctx) DcnvSVD(depths []float64, samples int, minPct float64) (sv []float64, removed int, err error) {
	n := len(depths) / samples
	sv = make([]float64, samples)
	var nr C.int32_t
	rc := C.gl_dcnv_svd(c.h, (*C.double)(&depths[0]), C.int64_t(n), C.int64_t(samples), C.int32_t(samples), C.double(minPct), 0,
		(*C.double)(&sv[0]), nil, &nr, nil)
	return sv, int(nr), c.err(rc)
}

// FormatF2 is fmt.Sprintf("%.2f", v) of every value, made on the GPU: 16 bytes per value, the text NUL-padded; an empty
// token means the text is longer and the caller formats that value itself.
func (c *Ctx) FormatF2(vals []float64) ([]byte, error) {
	tok := make([]byte, 16*len(vals)+16)
	rc := C.gl_format_f2(c.h, (*C.double)(&vals[0]), C.int64_t(len(vals)), (*C.uint8_t)(&tok[0]))
	return tok[:16*len(vals)], c.err(rc)
}

// Emdepth replaces emdepth.EMDepth + EMD.CN / Log2FC / Same of emdepth/emdepth.go:117-304 on the n x S row-major float32
// matrix `depths`: one byte per cell (bits 0-3 the CN, bits 4-5 the Same class of Log2FC, bit 6 set when Log2FC is outside
// (-0.5, 0.3)), and the nine final centres of every row.  Rows are streamed in blocks sized to free device memory.
func (c *Ctx) Emdepth(depths []float32, samples int) (cells []uint8, lambda []float64, err error) {
	n := len(depths) / samples
	cells = make([]uint8, n*samples+1)
	lambda = make([]float64, n*9+1)
	rc := C.gl_emdepth(c.h, (*C.float)(&depths[0]), C.int64_t(n), C.int64_t(samples), C.int32_t(samples), 0,
		(*C.uint8_t)(&cells[0]), (*C.double)(&lambda[0]))
	return cells[:n*samples], lambda[:n*9], c.err(rc)
}

// CNVCall is one test-set call: the sample's index, the chromosome's rank in bytewise name order, start, end and CN.
type CNVCall struct {
	Sample, Chrom  int32
	Start, End, CN int64
}

// CNVTruth is one truth-set site: the chromosome's rank, start, end, CN and the samples that carry it (a sample listed
// twice counts twice).
type CNVTruth struct {
	Chrom          int32
	Start, End, CN int64
	Samples        []int32
}

// CNVEval replaces cnveval.Evaluate (cnveval/cnveval.go:163-341) for calls in file order: stats[s*12 + class*4 + k] is
// the count k (TP, FP, FN, TN) of sample s in size class 0 (< 20000), 1 (< 100000) or 2, the reference's CohortStats.
// Each sample's calls are put in Go's sort.Slice order on the host; the comparison runs on the GPU (DESIGN §1.12).
func (c *Ctx) CNVEval(samples int, calls []CNVCall, truths []CNVTruth, minOverlap float64) ([]uint64, error) {
	nc, nt := len(calls), len(truths)
	cs, cc := make([]int32, nc+1), make([]int32, nc+1)
	cb, ce, ccn := make([]int64, nc+1), make([]int64, nc+1), make([]int64, nc+1)
	for i, x := range calls {
		cs[i], cc[i], cb[i], ce[i], ccn[i] = x.Sample, x.Chrom, x.Start, x.End, x.CN
	}
	tc, mp := make([]int32, nt+1), make([]int64, nt+1)
	tb, te, tcn := make([]int64, nt+1), make([]int64, nt+1), make([]int64, nt+1)
	ms := make([]int32, 0, nt+1)
	for i, t := range truths {
		tc[i], tb[i], te[i], tcn[i] = t.Chrom, t.Start, t.End, t.CN
		ms = append(ms, t.Samples...)
		mp[i+1] = int64(len(ms))
	}
	ms = append(ms, 0)
	stats := make([]uint64, samples*12+1)
	rc := C.gl_cnveval(c.h, C.int32_t(samples), (*C.int32_t)(&cs[0]), (*C.int32_t)(&cc[0]), (*C.int64_t)(&cb[0]),
		(*C.int64_t)(&ce[0]), (*C.int64_t)(&ccn[0]), C.int64_t(nc), (*C.int32_t)(&tc[0]), (*C.int64_t)(&tb[0]),
		(*C.int64_t)(&te[0]), (*C.int64_t)(&tcn[0]), C.int64_t(nt), (*C.int64_t)(&mp[0]), (*C.int32_t)(&ms[0]),
		C.double(minOverlap), (*C.uint64_t)(&stats[0]))
	return stats[:samples*12], c.err(rc)
}

// IndexcovPCA replaces indexcov's pca (indexcov/indexcov.go:773-807) on the samples x d byte matrix x (row-major, one row
// of PCA bytes per sample): the projections X V[:, :k] (samples x k, row-major) for k = min(5, samples, d), with the sign
// and rank rules of DESIGN §1.11, and the singular values.  The Gram runs on the tensor cores.
func (c *Ctx) IndexcovPCA(x []uint8, samples int) (proj []float64, sv []float64, k int, err error) {
	if samples < 1 || len(x) < samples || len(x)%samples != 0 {
		return nil, nil, 0, fmt.Errorf("IndexcovPCA: %d bytes are not %d rows", len(x), samples)
	}
	d := len(x) / samples
	proj = make([]float64, samples*5)
	sv = make([]float64, 5)
	var ko C.int32_t
	rc := C.gl_indexcov_pca(c.h, (*C.uint8_t)(&x[0]), C.int64_t(d), C.int32_t(samples), C.int64_t(d), 5,
		(*C.double)(&proj[0]), (*C.double)(&sv[0]), &ko, nil)
	if err = c.err(rc); err != nil {
		return nil, nil, 0, err
	}
	k = int(ko)
	out := make([]float64, samples*k)
	for i := 0; i < samples; i++ {
		copy(out[i*k:(i+1)*k], proj[i*5:i*5+k])
	}
	return out, sv[:k], k, nil
}

// EmdepthStats reports, for the last Emdepth call, the rows done, the cells decided inside the error band of the
// reference's CPU-dependent Exp / Log, and the bin means summed in sample order.
func (c *Ctx) EmdepthStats() (rows, uncertified, sequential int64) {
	var r, u, s C.int64_t
	C.gl_emdepth_stats(c.h, &r, &u, &s)
	return int64(r), int64(u), int64(s)
}

// EmdepthCNV is one emdepth.CNV: the sample, PSize, and the rows it holds (their CNs are cells[row*S+Sample] & 15).
type EmdepthCNV struct {
	Sample, PSize int
	Rows          []int64
}

// EmdepthCNVs walks emdepth.Cache over the cells in row order (emdepth/emdepth.go:330-398), with Clear(nil) before every
// row in breaks (the rows where a chromosome starts) and after the last row.  CNVs of one Clear come in sample order.
func EmdepthCNVs(cells []uint8, samples int, starts, ends, breaks []int64) ([]EmdepthCNV, error) {
	n := len(starts)
	var nc, nr C.int64_t
	pc := (*C.uint8_t)(unsafe.Pointer(nil))
	if len(cells) > 0 {
		pc = (*C.uint8_t)(&cells[0])
	}
	ps, pe, pb := (*C.int64_t)(unsafe.Pointer(nil)), (*C.int64_t)(unsafe.Pointer(nil)), (*C.int64_t)(unsafe.Pointer(nil))
	if n > 0 {
		ps, pe = (*C.int64_t)(&starts[0]), (*C.int64_t)(&ends[0])
	}
	if len(breaks) > 0 {
		pb = (*C.int64_t)(&breaks[0])
	}
	if C.gl_emdepth_cnvs(pc, C.int64_t(n), C.int32_t(samples), ps, pe, pb, C.int64_t(len(breaks)), nil, nil, nil, 0, &nc,
		nil, 0, &nr) != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: gl_emdepth_cnvs failed")
	}
	smp, psz := make([]int32, nc+1), make([]int32, nc+1)
	ptr, rows := make([]int64, nc+1), make([]int64, nr+1)
	if C.gl_emdepth_cnvs(pc, C.int64_t(n), C.int32_t(samples), ps, pe, pb, C.int64_t(len(breaks)), (*C.int32_t)(&smp[0]),
		(*C.int32_t)(&psz[0]), (*C.int64_t)(&ptr[0]), nc, &nc, (*C.int64_t)(&rows[0]), nr, &nr) != C.GL_OK {
		return nil, fmt.Errorf("goleft_b200: gl_emdepth_cnvs failed")
	}
	out := make([]EmdepthCNV, int(nc))
	for i := range out {
		out[i] = EmdepthCNV{Sample: int(smp[i]), PSize: int(psz[i]), Rows: append([]int64(nil), rows[ptr[i]:ptr[i+1]]...)}
	}
	return out, nil
}

// Stats is covstats.Stats (covstats/covstats.go:92-112) as gl_bam_covstats computes it.
type Stats struct {
	InsertMean, InsertSD                 float64
	InsertPct5, InsertPct95              int
	TemplateMean, TemplateSD             float64
	ReadLengthMean, ReadLengthMedian     float64
	ProportionBad, ProportionUnmapped    float64
	ProportionProperlyPaired             float64
	ProportionDuplicate                  float64
	MaxReadLength                        int
	H                                    []float64
	// OnDevice tells whether the records were sampled on the GPU (false: the file went through the host sampler)
	OnDevice bool
	// Prefetched tells whether the first batch came from PrefetchBamStats
	Prefetched bool
}

// PrefetchBamStats starts reading the first batch of next for a later BamStats(next, n, skipReads) on this Ctx and returns at
// once, so that the read overlaps the BAM sampled before it.  A file the GPU would refuse gets no prefetch (BamStats then
// takes the host sampler); the prefetch is dropped when next is closed or another prefetch starts.
func (c *Ctx) PrefetchBamStats(next *Bam, n, skipReads int) error {
	return c.err(C.gl_bam_covstats_prefetch(c.h, next.h, C.int32_t(n), C.int32_t(skipReads)))
}

// BamStats replaces covstats.BamStats(br, n, skipReads) (covstats/covstats.go:122-220): the records are sampled on the
// GPU, or by the host sampler when the file cannot be taken there (GL_ESTATE: no index, a BGZF member the device rejects).
// Where the reference panics (1 or 2 insert sizes, a negative histogram length) it returns the library's error.
func (c *Ctx) BamStats(b *Bam, n, skipReads int) (Stats, error) {
	var st C.gl_covstats
	h := make([]float64, 1<<14)
	call := func(device bool) C.int {
		for {
			var rc C.int
			if device {
				rc = C.gl_bam_covstats(c.h, b.h, C.int32_t(n), C.int32_t(skipReads), &st, (*C.double)(unsafe.Pointer(&h[0])), C.int64_t(len(h)))
			} else {
				rc = C.gl_bam_covstats_host(c.h, b.h, C.int32_t(n), C.int32_t(skipReads), &st, (*C.double)(unsafe.Pointer(&h[0])), C.int64_t(len(h)))
			}
			if rc == C.GL_ERANGE && int(st.h_len) > len(h) {
				h = make([]float64, int(st.h_len))
				continue
			}
			return rc
		}
	}
	rc := call(true)
	if rc == C.GL_ESTATE {
		rc = call(false)
	}
	if e := c.err(rc); e != nil {
		return Stats{}, e
	}
	return Stats{
		InsertMean: float64(st.insert_mean), InsertSD: float64(st.insert_sd), InsertPct5: int(st.insert_pct5), InsertPct95: int(st.insert_pct95),
		TemplateMean: float64(st.template_mean), TemplateSD: float64(st.template_sd),
		ReadLengthMean: float64(st.read_length_mean), ReadLengthMedian: float64(st.read_length_median),
		ProportionBad: float64(st.proportion_bad), ProportionUnmapped: float64(st.proportion_unmapped),
		ProportionProperlyPaired: float64(st.proportion_properly_paired), ProportionDuplicate: float64(st.proportion_duplicate),
		MaxReadLength: int(st.max_read_length), H: h[:int(st.h_len)], OnDevice: st.path == 1, Prefetched: st.prefetched == 1,
	}, nil
}
