/* bamsynth.c — writes a coordinate-sorted BAM + BAI holding the reads of glsynth_core.h (ALL of them: duplicates, QC
 * fails, MAPQ 0 ... so a decoder's `samtools depth` filter has something to filter), for bench.py's CLI wall-clock leg
 * and the feeder tests.  WORKLOAD GENERATOR, not part of the depth engine.
 *
 * Layout like a real short-read BAM: 150-base reads with 4-bit sequence and one quality byte per base, BGZF blocks of
 * 0xff00 uncompressed bytes that records straddle freely, deflate level 1.  Three parallel passes over 32 KB cells:
 *   1. size   : bytes of BAM records per cell -> offset of every cell in the uncompressed stream
 *   2. deflate: workers take runs of 64 blocks, regenerate the cells under them, compress
 *   3. index  : virtual offset of every record -> bins + 16 KB linear index + the 37450 stats bin (SAM spec 5.2)
 * then the compressed blocks are written in order.
 *   gls_write_bam(path, n_contigs, names[], lengths[], seed_index[], coverage, read_len, threads) -> 0 / -1      (path.bai)
 *   gls_write_bam_csi(the same arguments)                                                                       (path.csi)
 * The CSI (CSIv1, min_shift 14, depth 5) holds the BAI's bins and chunks, each bin's loffset the 16 KB linear index at
 * the bin's first tile, the stats as the pseudo-bin 37450, BGZF-compressed.                                        */
#define _GNU_SOURCE
#include <pthread.h>
#include <stdio.h>
#include <zlib.h>
#include "glsynth_core.h"

#define BLK 0xff00
#define RUN_BLOCKS 64

typedef struct { uint8_t* p; size_t len, cap; } bbuf;
static void bb_put(bbuf* b, const void* src, size_t n) {
    if (b->len + n > b->cap) { b->cap = (b->len + n) * 2 + 4096; b->p = (uint8_t*)realloc(b->p, b->cap); }
    memcpy(b->p + b->len, src, n); b->len += n;
}
static void put32(bbuf* b, uint32_t v) { uint8_t t[4] = {(uint8_t)v, (uint8_t)(v >> 8), (uint8_t)(v >> 16), (uint8_t)(v >> 24)}; bb_put(b, t, 4); }

static int reg2bin(int64_t beg, int64_t end) {
    --end;
    if (beg >> 14 == end >> 14) return (int)(((1 << 15) - 1) / 7 + (beg >> 14));
    if (beg >> 17 == end >> 17) return (int)(((1 << 12) - 1) / 7 + (beg >> 17));
    if (beg >> 20 == end >> 20) return (int)(((1 << 9) - 1) / 7 + (beg >> 20));
    if (beg >> 23 == end >> 23) return (int)(((1 << 6) - 1) / 7 + (beg >> 23));
    if (beg >> 26 == end >> 26) return (int)(((1 << 3) - 1) / 7 + (beg >> 26));
    return 0;
}

/* cigar of a read -> ops (len<<4|op), reference span */
static int read_cigar(const gls_read* r, int L, uint32_t* cig, int* ref_span) {
    switch (r->kind) {
    case 1: cig[0] = ((uint32_t)r->k << 4) | 0; cig[1] = ((uint32_t)r->x << 4) | 2; cig[2] = ((uint32_t)(L - r->k) << 4) | 0; *ref_span = L + r->x; return 3;
    case 2: {
        int k = r->k; if (k > L - r->x - 1) k = L - r->x - 1; if (k < 1) k = 1;
        cig[0] = ((uint32_t)k << 4) | 0; cig[1] = ((uint32_t)r->x << 4) | 1; cig[2] = ((uint32_t)(L - k - r->x) << 4) | 0; *ref_span = L - r->x; return 3; }
    case 3: cig[0] = ((uint32_t)r->k << 4) | 4; cig[1] = ((uint32_t)(L - r->k) << 4) | 0; *ref_span = L - r->k; return 2;
    default: cig[0] = ((uint32_t)L << 4) | 0; *ref_span = L; return 1;
    }
}

static size_t record_size(const gls_read* r, int L, int64_t cell) {
    char name[40];
    const int ln = snprintf(name, sizeof name, "s%llx.%x", (unsigned long long)cell, r->id) + 1;
    uint32_t cig[3]; int span;
    const int nc = read_cigar(r, L, cig, &span);
    return 4 + 32 + (size_t)ln + 4u * (size_t)nc + (size_t)((L + 1) / 2) + (size_t)L;
}

static void write_record(bbuf* b, const gls_read* r, int L, int64_t cell, int tid, uint64_t seed) {
    char name[40];
    const int ln = snprintf(name, sizeof name, "s%llx.%x", (unsigned long long)cell, r->id) + 1;
    uint32_t cig[3]; int span;
    const int nc = read_cigar(r, L, cig, &span);
    const uint32_t bs = 32u + (uint32_t)ln + 4u * (uint32_t)nc + (uint32_t)((L + 1) / 2) + (uint32_t)L;
    put32(b, bs);
    put32(b, (uint32_t)tid); put32(b, (uint32_t)r->pos);
    const int bin = reg2bin(r->pos, (r->flag & 4) ? r->pos + 1 : r->pos + span);
    put32(b, (uint32_t)ln | ((uint32_t)r->mapq << 8) | ((uint32_t)bin << 16));
    put32(b, (uint32_t)nc | ((uint32_t)r->flag << 16));
    put32(b, (uint32_t)L);
    put32(b, 0xffffffffu); put32(b, 0xffffffffu); put32(b, 0);           /* next_refID -1, next_pos -1, tlen 0 */
    bb_put(b, name, (size_t)ln);
    for (int k = 0; k < nc; k++) put32(b, cig[k]);
    uint8_t seq[256];
    uint64_t h = gls_mix(seed ^ ((uint64_t)cell << 24) ^ r->id);
    for (int k = 0; k < (L + 1) / 2; k++) {                               /* 4-bit bases A C G T = 1 2 4 8 */
        if ((k & 15) == 0) h = gls_mix(h);
        const unsigned two = (unsigned)(h >> ((k & 15) * 4)) & 15u;
        seq[k] = (uint8_t)(((1u << (two & 3)) << 4) | (1u << (two >> 2)));
    }
    bb_put(b, seq, (size_t)((L + 1) / 2));
    uint8_t q[512];
    for (int k = 0; k < L; k++) q[k] = (uint8_t)(k < 8 || k > L - 20 ? 20 : 37);     /* binned qualities compress like real data */
    bb_put(b, q, (size_t)L);
}

typedef struct { uint64_t beg, end; } chunk_t;
typedef struct { int bin; chunk_t* ch; int n, cap; } bin_t;

typedef struct {
    int n_contigs; const char** names; const int64_t* lengths; gls_contig* C; int read_len;
    int64_t* cell_base;           /* [n_contigs+1] first global cell of each contig */
    int64_t n_cells;              /* total */
    int64_t* cell_off;            /* [n_cells+1] byte offset of each cell's records in the uncompressed stream */
    int64_t header_len; uint8_t* header;
    int64_t n_blocks; uint8_t** cblk; uint32_t* clen; int64_t* coff;   /* compressed blocks */
    int pass; int64_t next; pthread_mutex_t mu;
    int64_t* cell_reads;          /* [n_cells] for the index pass */
} BJob;

static int contig_of_cell(const BJob* J, int64_t gc) {
    int lo = 0, hi = J->n_contigs - 1;
    while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (J->cell_base[mid] <= gc) lo = mid; else hi = mid - 1; }
    return lo;
}

static size_t bgzf_compress_block(const uint8_t* in, size_t n, uint8_t* out) {
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    deflateInit2(&zs, 1, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY);
    zs.next_in = (Bytef*)in; zs.avail_in = (uInt)n;
    zs.next_out = out + 18; zs.avail_out = 0x10000 + 64 - 18 - 8;
    deflate(&zs, Z_FINISH);
    const size_t clen = zs.total_out;
    deflateEnd(&zs);
    const uint8_t hdr[18] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0, 0};
    memcpy(out, hdr, 18);
    const size_t bsize = 18 + clen + 8;
    out[16] = (uint8_t)((bsize - 1) & 0xff); out[17] = (uint8_t)((bsize - 1) >> 8);
    const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), in, (uInt)n), isz = (uint32_t)n;
    for (int i = 0; i < 4; i++) { out[18 + clen + i] = (uint8_t)(crc >> (8 * i)); out[22 + clen + i] = (uint8_t)(isz >> (8 * i)); }
    return bsize;
}

static void* bworker(void* arg) {
    BJob* J = (BJob*)arg;
    gls_read* rd = (gls_read*)malloc(sizeof(gls_read) * GLS_MAX_CELL_READS);
    uint64_t* pk = (uint64_t*)malloc(8 * (size_t)GLS_MAX_CELL_READS);
    bbuf raw = {0};
    for (;;) {
        pthread_mutex_lock(&J->mu);
        const int64_t w0 = J->next;
        J->next += (J->pass == 0 ? 64 : 1);
        pthread_mutex_unlock(&J->mu);
        if (J->pass == 0) {                                       /* sizes of 64 cells */
            if (w0 >= J->n_cells) break;
            for (int64_t gc = w0; gc < w0 + 64 && gc < J->n_cells; gc++) {
                const int t = contig_of_cell(J, gc);
                const int64_t m = gls_cell_reads(&J->C[t], gc - J->cell_base[t], rd, pk);
                int64_t bytes = 0;
                for (int64_t j = 0; j < m; j++) bytes += (int64_t)record_size(&rd[j], J->read_len, gc - J->cell_base[t]);
                J->cell_off[gc + 1] = bytes;
                J->cell_reads[gc] = m;
            }
        } else {                                                  /* compress one run of blocks */
            const int64_t b0 = w0 * RUN_BLOCKS;
            if (b0 >= J->n_blocks) break;
            const int64_t b1 = b0 + RUN_BLOCKS < J->n_blocks ? b0 + RUN_BLOCKS : J->n_blocks;
            const int64_t total = J->header_len + J->cell_off[J->n_cells];
            const int64_t s0 = b0 * BLK, s1 = b1 * BLK < total ? b1 * BLK : total;      /* stream range of the run */
            raw.len = 0;
            int64_t at = s0;                                      /* stream offset of raw.p[0] */
            if (s0 < J->header_len) {
                const int64_t h1 = s1 < J->header_len ? s1 : J->header_len;
                bb_put(&raw, J->header + s0, (size_t)(h1 - s0));
            }
            /* cells overlapping [max(s0,header), s1) */
            const int64_t r0 = (s0 > J->header_len ? s0 : J->header_len) - J->header_len, r1 = s1 - J->header_len;
            if (r1 > r0) {
                int64_t lo = 0, hi = J->n_cells;                  /* first cell with cell_off[c+1] > r0 */
                while (lo < hi) { int64_t mid = (lo + hi) >> 1; if (J->cell_off[mid + 1] > r0) hi = mid; else lo = mid + 1; }
                int64_t gc = lo;
                int64_t skip = r0 - J->cell_off[gc];              /* bytes of the first cell that belong to the previous run */
                for (; gc < J->n_cells && J->cell_off[gc] < r1; gc++) {
                    const int t = contig_of_cell(J, gc);
                    const int64_t m = gls_cell_reads(&J->C[t], gc - J->cell_base[t], rd, pk);
                    bbuf cell = {0};
                    for (int64_t j = 0; j < m; j++) write_record(&cell, &rd[j], J->read_len, gc - J->cell_base[t], t, J->C[t].seed);
                    int64_t take0 = skip, take1 = (int64_t)cell.len;
                    if (J->cell_off[gc] + take1 > r1) take1 = r1 - J->cell_off[gc];
                    if (take1 > take0) bb_put(&raw, cell.p + take0, (size_t)(take1 - take0));
                    free(cell.p);
                    skip = 0;
                }
            }
            (void)at;
            for (int64_t b = b0; b < b1; b++) {
                const int64_t o = (b - b0) * BLK;
                const int64_t n = (int64_t)raw.len - o < BLK ? (int64_t)raw.len - o : BLK;
                uint8_t* out = (uint8_t*)malloc(0x10000 + 64);
                J->clen[b] = (uint32_t)bgzf_compress_block(raw.p + o, (size_t)(n > 0 ? n : 0), out);
                J->cblk[b] = out;
            }
        }
    }
    free(rd); free(pk); free(raw.p);
    return NULL;
}

static void brun(BJob* J, int threads) {
    pthread_t th[256];
    if (threads > 256) threads = 256;
    if (threads < 1) threads = 1;
    J->next = 0;
    for (int t = 1; t < threads; t++) pthread_create(&th[t], NULL, bworker, J);
    bworker(J);
    for (int t = 1; t < threads; t++) pthread_join(th[t], NULL);
}

static int cmp_bin(const void* a, const void* b) { return ((const bin_t*)a)->bin - ((const bin_t*)b)->bin; }

static int write_bam(const char* path, int n_contigs, const char** names, const int64_t* lengths, const int* seed_index,
                     double coverage, int read_len, int threads, int csi) {
    if (n_contigs <= 0 || read_len < 20 || read_len > 250) return -1;
    BJob J;
    memset(&J, 0, sizeof J);
    J.n_contigs = n_contigs; J.names = names; J.lengths = lengths; J.read_len = read_len;
    J.C = (gls_contig*)calloc((size_t)n_contigs, sizeof(gls_contig));
    J.cell_base = (int64_t*)calloc((size_t)n_contigs + 1, 8);
    for (int t = 0; t < n_contigs; t++) {
        gls_contig_init(&J.C[t], lengths[t], coverage, read_len, 0x601EF7ull + (uint64_t)seed_index[t], 1, 1);
        J.cell_base[t + 1] = J.cell_base[t] + J.C[t].n_cells;
    }
    J.n_cells = J.cell_base[n_contigs];
    J.cell_off = (int64_t*)calloc((size_t)J.n_cells + 1, 8);
    J.cell_reads = (int64_t*)calloc((size_t)J.n_cells + 1, 8);
    /* header */
    bbuf h = {0};
    bbuf text = {0};
    const char* hd = "@HD\tVN:1.6\tSO:coordinate\n";
    bb_put(&text, hd, strlen(hd));
    for (int t = 0; t < n_contigs; t++) {
        char ln[256];
        const int n = snprintf(ln, sizeof ln, "@SQ\tSN:%s\tLN:%lld\n", names[t], (long long)lengths[t]);
        bb_put(&text, ln, (size_t)n);
    }
    const char* rg = "@RG\tID:synth\tSM:synth30x\n";
    bb_put(&text, rg, strlen(rg));
    bb_put(&h, "BAM\1", 4); put32(&h, (uint32_t)text.len); bb_put(&h, text.p, text.len); put32(&h, (uint32_t)n_contigs);
    for (int t = 0; t < n_contigs; t++) { put32(&h, (uint32_t)strlen(names[t]) + 1); bb_put(&h, names[t], strlen(names[t]) + 1); put32(&h, (uint32_t)lengths[t]); }
    J.header = h.p; J.header_len = (int64_t)h.len;
    pthread_mutex_init(&J.mu, NULL);
    J.pass = 0; brun(&J, threads);
    for (int64_t c = 0; c < J.n_cells; c++) J.cell_off[c + 1] += J.cell_off[c];
    const int64_t total = J.header_len + J.cell_off[J.n_cells];
    J.n_blocks = (total + BLK - 1) / BLK;
    J.cblk = (uint8_t**)calloc((size_t)J.n_blocks + 1, sizeof(uint8_t*));
    J.clen = (uint32_t*)calloc((size_t)J.n_blocks + 1, 4);
    J.coff = (int64_t*)calloc((size_t)J.n_blocks + 2, 8);
    J.pass = 1; brun(&J, threads);
    for (int64_t b = 0; b < J.n_blocks; b++) J.coff[b + 1] = J.coff[b] + J.clen[b];
    FILE* f = fopen(path, "wb");
    if (!f) return -1;
    for (int64_t b = 0; b < J.n_blocks; b++) { fwrite(J.cblk[b], 1, J.clen[b], f); free(J.cblk[b]); }
    static const uint8_t eof_blk[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    fwrite(eof_blk, 1, 28, f);
    fclose(f);

    /* ---- index: sequential over records (sizes only; cheap next to the deflate pass) */
    char ipath[4096];
    snprintf(ipath, sizeof ipath, csi ? "%s.csi" : "%s.bai", path);
    FILE* fi = fopen(ipath, "wb");
    if (!fi) return -1;
    bbuf ix = {0};
    if (csi) { bb_put(&ix, "CSI\1", 4); put32(&ix, 14); put32(&ix, 5); put32(&ix, 0); }     /* min_shift, depth, l_aux */
    else bb_put(&ix, "BAI\1", 4);
    put32(&ix, (uint32_t)n_contigs);
    gls_read* rd = (gls_read*)malloc(sizeof(gls_read) * GLS_MAX_CELL_READS);
    uint64_t* pk = (uint64_t*)malloc(8 * (size_t)GLS_MAX_CELL_READS);
#define VOFF(so) ((((uint64_t)J.coff[(so) / BLK]) << 16) | (uint64_t)((so) % BLK))
    for (int t = 0; t < n_contigs; t++) {
        const int64_t n_tiles = (lengths[t] + 16383) >> 14;
        uint64_t* lin = (uint64_t*)calloc((size_t)n_tiles + 1, 8);
        int64_t lin_n = 0;
        bin_t* bins = NULL; int nbins = 0, capbins = 0;
        int* bin_slot = (int*)malloc(sizeof(int) * 37450);
        for (int k = 0; k < 37450; k++) bin_slot[k] = -1;
        uint64_t n_mapped = 0, n_unmapped = 0, ref_beg = 0, ref_end = 0;
        int have = 0;
        int last_bin = -1;
        for (int64_t lc = 0; lc < J.C[t].n_cells; lc++) {
            const int64_t gc = J.cell_base[t] + lc;
            if (J.cell_reads[gc] == 0) continue;
            const int64_t m = gls_cell_reads(&J.C[t], lc, rd, pk);
            int64_t so = J.header_len + J.cell_off[gc];
            for (int64_t j = 0; j < m; j++) {
                const gls_read* r = &rd[j];
                uint32_t cig[3]; int span;
                read_cigar(r, read_len, cig, &span);
                const int64_t rs = (int64_t)record_size(r, read_len, lc);
                const uint64_t v0 = VOFF(so), v1 = VOFF(so + rs);
                const int64_t beg = r->pos, end = (r->flag & 4) ? r->pos + 1 : r->pos + span;
                const int bin = reg2bin(beg, end);
                if (!have) { ref_beg = v0; have = 1; }
                ref_end = v1;
                if (r->flag & 4) n_unmapped++; else n_mapped++;
                if (bin_slot[bin] < 0) {
                    if (nbins == capbins) { capbins = capbins * 2 + 64; bins = (bin_t*)realloc(bins, sizeof(bin_t) * (size_t)capbins); }
                    bins[nbins].bin = bin; bins[nbins].ch = NULL; bins[nbins].n = bins[nbins].cap = 0;
                    bin_slot[bin] = nbins++;
                }
                bin_t* B = &bins[bin_slot[bin]];
                if (bin == last_bin && B->n > 0) B->ch[B->n - 1].end = v1;          /* consecutive records of one bin: one chunk */
                else {
                    if (B->n == B->cap) { B->cap = B->cap * 2 + 4; B->ch = (chunk_t*)realloc(B->ch, sizeof(chunk_t) * (size_t)B->cap); }
                    B->ch[B->n].beg = v0; B->ch[B->n].end = v1; B->n++;
                }
                last_bin = bin;
                for (int64_t k = beg >> 14; k <= (end - 1) >> 14 && k < n_tiles; k++) {
                    if (lin[k] == 0) lin[k] = v0;                                    /* records come in file order: the first is the smallest */
                    if (k + 1 > lin_n) lin_n = k + 1;
                }
                so += rs;
            }
        }
        for (int64_t k = lin_n - 2; k >= 0; k--) if (lin[k] == 0) lin[k] = lin[k + 1];   /* htslib back-fills empty tiles */
        qsort(bins, (size_t)nbins, sizeof(bin_t), cmp_bin);
        put32(&ix, (uint32_t)(nbins + (have ? 1 : 0)));
        for (int k = 0; k < nbins; k++) {
            put32(&ix, (uint32_t)bins[k].bin);
            if (csi) {                                                       /* loffset: the linear index at the bin's first tile */
                static const int first[6] = {0, 1, 9, 73, 585, 4681};
                int l = 5;
                while (bins[k].bin < first[l]) l--;
                const int64_t bot = (int64_t)(bins[k].bin - first[l]) << (3 * (5 - l));
                const uint64_t lo = bot < lin_n ? lin[bot] : 0;
                put32(&ix, (uint32_t)lo); put32(&ix, (uint32_t)(lo >> 32));
            }
            put32(&ix, (uint32_t)bins[k].n);
            for (int c = 0; c < bins[k].n; c++) { put32(&ix, (uint32_t)bins[k].ch[c].beg); put32(&ix, (uint32_t)(bins[k].ch[c].beg >> 32)); put32(&ix, (uint32_t)bins[k].ch[c].end); put32(&ix, (uint32_t)(bins[k].ch[c].end >> 32)); }
            free(bins[k].ch);
        }
        if (have) {
            put32(&ix, 37450);
            if (csi) { put32(&ix, 0); put32(&ix, 0); }
            put32(&ix, 2);
            const uint64_t q[4] = {ref_beg, ref_end, n_mapped, n_unmapped};
            for (int k = 0; k < 4; k++) { put32(&ix, (uint32_t)q[k]); put32(&ix, (uint32_t)(q[k] >> 32)); }
        }
        if (!csi) {                                                          /* a CSI has no linear index */
            put32(&ix, (uint32_t)lin_n);
            for (int64_t k = 0; k < lin_n; k++) { put32(&ix, (uint32_t)lin[k]); put32(&ix, (uint32_t)(lin[k] >> 32)); }
        }
        free(lin); free(bins); free(bin_slot);
    }
    put32(&ix, 0); put32(&ix, 0);                                    /* n_no_coor */
    if (csi) {                                                       /* BGZF, then the EOF block */
        uint8_t* out = (uint8_t*)malloc(0x10000 + 64);
        for (size_t o = 0; o < ix.len; o += BLK) fwrite(out, 1, bgzf_compress_block(ix.p + o, ix.len - o < BLK ? ix.len - o : BLK, out), fi);
        fwrite(out, 1, bgzf_compress_block(NULL, 0, out), fi);
        free(out);
    } else {
        fwrite(ix.p, 1, ix.len, fi);
    }
    fclose(fi);
    free(ix.p); free(rd); free(pk); free(h.p); free(text.p);
    free(J.C); free(J.cell_base); free(J.cell_off); free(J.cell_reads); free(J.cblk); free(J.clen); free(J.coff);
    pthread_mutex_destroy(&J.mu);
    return 0;
}

int gls_write_bam(const char* path, int n_contigs, const char** names, const int64_t* lengths, const int* seed_index,
                  double coverage, int read_len, int threads) {
    return write_bam(path, n_contigs, names, lengths, seed_index, coverage, read_len, threads, 0);
}

int gls_write_bam_csi(const char* path, int n_contigs, const char** names, const int64_t* lengths, const int* seed_index,
                      double coverage, int read_len, int threads) {
    return write_bam(path, n_contigs, names, lengths, seed_index, coverage, read_len, threads, 1);
}
