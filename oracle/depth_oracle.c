/*
 * depth_oracle.c -- TEST INFRASTRUCTURE ONLY.  Not part of the product path.
 *
 * A single-threaded CPU restatement of the `sambamba depth {base,region,window}`
 * algorithm, used as the parity checker for the CUDA engine in sambamba_b200/.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may build, link or execute this file.
 *
 * The reference (biod/sambamba @ v1.0.1) is D and cannot be compiled in this
 * image (no ldc2/dmd/gdc), so this is a "port" oracle.  It is pinned against
 * the reference's own golden files (tests/golden/, copied from
 * the reference's test/ directory): issue_193, issue225 (-c 1 / -c 0, with and without
 * -L chrM) and issue_204 (region -T x3 -m).  See tests/test_oracle_golden.py.
 *
 * Third-party arithmetic: raw DEFLATE inflate lives in system zlib, exactly as
 * in the reference (BioD/bio/core/utils/zlib.d:6, block.d:162-183 call
 * inflateInit2(-15)/inflate(Z_FINISH)/inflateEnd).  The oracle calls the same
 * library.
 *
 * Each section cites the reference file:line it follows (paths relative to
 * biod/sambamba v1.0.1).  Nothing here is copied from the reference; it is C
 * restating D semantics.
 *
 * Build:  make -C oracle     (-> oracle/_build/depth_oracle, liboracle.so)
 */
#define _GNU_SOURCE
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdarg.h>
#include <math.h>
#include <pthread.h>
#include <stdatomic.h>
#include <zlib.h>

/* ------------------------------------------------------------------ utils */

static char g_err[1024];
static int fail(const char *fmt, ...) {
    va_list ap; va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return -1;
}
const char *oracle_last_error(void) { return g_err; }

static uint16_t rd16(const uint8_t *p) { return (uint16_t)(p[0] | (p[1] << 8)); }
static uint32_t rd32(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
static uint64_t rd64(const uint8_t *p) { return (uint64_t)rd32(p) | ((uint64_t)rd32(p + 4) << 32); }

#define VEC_PUSH(arr, n, cap, val) do { \
    if ((n) == (cap)) { (cap) = (cap) ? (cap) * 2 : 16; (arr) = realloc((arr), (cap) * sizeof *(arr)); } \
    (arr)[(n)++] = (val); } while (0)

/* ---------------------------------------------------------- BGZF (layer 1)
 * Block framing: BioD/bio/core/bgzf/inputstream.d:54-199 (fillBgzfBufferFromStream)
 * constants:     BioD/bio/core/bgzf/constants.d:26-61
 * inflate:       BioD/bio/core/bgzf/block.d:127-216 (decompressBgzfBlock)
 * EOF handling:  inputstream.d:386-424 (fillNextBlock stops at input_size == 0)
 */
typedef struct {
    uint64_t coff;      /* offset of the block in the compressed file      */
    uint32_t cdata_off; /* offset of raw deflate data within the block     */
    uint32_t cdata_size;
    uint32_t bsize;     /* total block size                                */
    uint32_t isize;     /* uncompressed size                               */
    uint64_t uoff;      /* offset in the concatenated uncompressed stream  */
} BgzfBlock;

typedef struct {
    uint8_t *file; size_t file_len;
    BgzfBlock *blocks; size_t n_blocks, cap_blocks;
    uint8_t *u; size_t ulen;      /* concatenated inflated payload */
    int sampled;                  /* --max-file-bytes cut the file (bench's bounded sample): the stream may end inside a record */
} Bgzf;

static int bgzf_index(Bgzf *z) {
    size_t off = 0; uint64_t uoff = 0;
    while (off < z->file_len) {
        const uint8_t *p = z->file + off;
        if (z->file_len - off < 4) break;                    /* inputstream.d:74-79: short read -> no block */
        if (!(p[0] == 0x1f && p[1] == 0x8b && p[2] == 0x08 && p[3] == 0x04))
            return fail("Error reading BGZF block starting from offset %zu: wrong BGZF magic", off);
        if (z->file_len - off < 12) return fail("Error reading BGZF block starting from offset %zu: stream error", off);
        uint32_t xlen = rd16(p + 10);
        if (z->file_len - off < 12 + xlen) return fail("Error reading BGZF block starting from offset %zu: stream error", off);
        uint32_t len = 0, bsize = 0; int found = 0;
        while (len < xlen) {
            if (len + 4 > xlen) break;
            uint8_t si1 = p[12 + len], si2 = p[13 + len]; uint32_t slen = rd16(p + 14 + len);
            if (si1 == 66 && si2 == 67) {
                if (slen != 2) return fail("Error reading BGZF block starting from offset %zu: wrong BC subfield length: %u; expected 2", off, slen);
                if (found) return fail("Error reading BGZF block starting from offset %zu: duplicate field with block size", off);
                bsize = rd16(p + 16 + len); found = 1;
            }
            len += 4 + slen;
        }
        if (len != xlen) return fail("Error reading BGZF block starting from offset %zu: total length of subfields in bytes (%u) is not equal to gzip_extra_length (%u)", off, len, xlen);
        if (!found) return fail("Error reading BGZF block starting from offset %zu: block size was not found in any subfield", off);
        int64_t cdata_size = (int64_t)bsize - xlen - 19;
        if (cdata_size < 0 || cdata_size > 65536) return fail("Error reading BGZF block starting from offset %zu: compressed data size is more than 65536 bytes, which is not allowed by current BAM specification", off);
        size_t total = (size_t)bsize + 1;
        if (z->file_len - off < total) return fail("Error reading BGZF block starting from offset %zu: stream error: not enough data in stream", off);
        uint32_t isize = rd32(p + total - 4);
        if (isize == 0) break;                                /* EOF marker / empty block ends the stream (inputstream.d:393) */
        if (isize > 65536) return fail("Error reading BGZF block starting from offset %zu: input size is more than 65536", off);
        BgzfBlock b = { off, 12 + xlen, (uint32_t)cdata_size, (uint32_t)total, isize, uoff };
        VEC_PUSH(z->blocks, z->n_blocks, z->cap_blocks, b);
        uoff += isize; off += total;
    }
    z->ulen = uoff;
    return 0;
}

static int inflate_block(const Bgzf *z, const BgzfBlock *b, uint8_t *dst) {
    z_stream zs; memset(&zs, 0, sizeof zs);
    zs.next_in = (Bytef *)(z->file + b->coff + b->cdata_off); zs.avail_in = b->cdata_size;
    zs.next_out = dst; zs.avail_out = b->isize;
    if (inflateInit2(&zs, -15) != Z_OK) return fail("zlib: inflateInit2 failed");
    int r = inflate(&zs, Z_FINISH);
    inflateEnd(&zs);
    if (r != Z_STREAM_END || zs.total_out != b->isize) return fail("zlib: inflate failed (block at %llu)", (unsigned long long)b->coff);
    return 0;
}

typedef struct { const Bgzf *z; size_t lo, hi; int rc; } InflateJob;
static void *inflate_worker(void *arg) {
    InflateJob *j = arg;
    for (size_t i = j->lo; i < j->hi; i++)
        if (inflate_block(j->z, &j->z->blocks[i], j->z->u + j->z->blocks[i].uoff)) { j->rc = -1; break; }
    return NULL;
}

/* Inflate every block.  nthreads mirrors the reference's only parallel stage
 * (task!decompressBgzfBlock on std.parallelism workers, inputstream.d:414-417). */
static int bgzf_inflate_all(Bgzf *z, int nthreads) {
    z->u = malloc(z->ulen ? z->ulen : 1);
    if (!z->u) return fail("out of memory");
    if (nthreads < 1) nthreads = 1;
    if ((size_t)nthreads > z->n_blocks) nthreads = z->n_blocks ? (int)z->n_blocks : 1;
    pthread_t *th = calloc(nthreads, sizeof *th); InflateJob *jobs = calloc(nthreads, sizeof *jobs);
    for (int t = 0; t < nthreads; t++) {
        jobs[t].z = z; jobs[t].lo = z->n_blocks * t / nthreads; jobs[t].hi = z->n_blocks * (t + 1) / nthreads;
        if (nthreads > 1) pthread_create(&th[t], NULL, inflate_worker, &jobs[t]); else inflate_worker(&jobs[t]);
    }
    int rc = 0;
    for (int t = 0; t < nthreads; t++) { if (nthreads > 1) pthread_join(th[t], NULL); if (jobs[t].rc) rc = -1; }
    free(th); free(jobs);
    return rc;
}

static int bgzf_load(Bgzf *z, const char *path, int nthreads, size_t max_file_bytes) {
    memset(z, 0, sizeof *z);
    FILE *f = fopen(path, "rb");
    if (!f) return fail("Cannot open file `%s' in mode `rb' (No such file or directory)", path);
    fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET);
    if (max_file_bytes && (size_t)n > max_file_bytes) n = (long)max_file_bytes;
    z->file = malloc(n ? n : 1); z->file_len = n;
    if (fread(z->file, 1, n, f) != (size_t)n) { fclose(f); return fail("read error"); }
    fclose(f);
    if (max_file_bytes) {
        /* bounded sample: keep only whole blocks */
        size_t off = 0;
        while (off + 18 <= z->file_len) { size_t t = (size_t)rd16(z->file + off + 16) + 1; if (off + t > z->file_len) break; off += t; }
        z->file_len = off; z->sampled = 1;
    }
    if (bgzf_index(z)) return -1;
    return bgzf_inflate_all(z, nthreads);
}
static void bgzf_free(Bgzf *z) { free(z->file); free(z->blocks); free(z->u); memset(z, 0, sizeof *z); }

/* ------------------------------------------------------ BAM header (layer 2)
 * magic / l_text / text / n_ref / refs: BioD/bio/std/hts/bam/reader.d:101-125,580-598
 * @HD SO, @RG ID/SM:                    BioD/bio/std/hts/sam/header.d:461-530
 * sample table:                         sambamba/depth.d:1170-1181
 */
typedef struct { char *name; uint32_t length; } RefSeq;
typedef struct {
    Bgzf z;
    int n_ref; RefSeq *refs;
    size_t first_rec;
    int so_coordinate;
    int n_samples; char **sample_names;
    int n_rg; char **rg_ids; int *rg_sample;
} Bam;

static char *dupn(const char *s, size_t n) { char *r = malloc(n + 1); memcpy(r, s, n); r[n] = 0; return r; }

static int bam_parse_header(Bam *b, int allow_truncated) {
    const uint8_t *u = b->z.u; size_t n = b->z.ulen;
    if (n < 12 || memcmp(u, "BAM\1", 4)) return fail("Invalid file format: expected BAM\\1");
    uint32_t l_text = rd32(u + 4);
    if (8 + (size_t)l_text + 4 > n) return fail("truncated BAM header");
    const char *text = (const char *)u + 8;
    size_t off = 8 + l_text;
    b->n_ref = (int)rd32(u + off); off += 4;
    b->refs = calloc(b->n_ref ? b->n_ref : 1, sizeof *b->refs);
    for (int i = 0; i < b->n_ref; i++) {
        if (off + 4 > n) return fail("truncated BAM header");
        uint32_t l_name = rd32(u + off); off += 4;
        if (off + l_name + 4 > n) return fail("truncated BAM header");
        b->refs[i].name = dupn((const char *)u + off, l_name ? l_name - 1 : 0); off += l_name;
        b->refs[i].length = rd32(u + off); off += 4;
    }
    b->first_rec = off;
    (void)allow_truncated;
    /* SAM header text: one line per record, tab separated TAG:VALUE fields */
    size_t p = 0;
    while (p < l_text) {
        size_t e = p; while (e < l_text && text[e] != '\n') e++;
        if (e - p >= 3 && text[p] == '@') {
            int is_hd = !strncmp(text + p, "@HD", 3), is_rg = !strncmp(text + p, "@RG", 3);
            if (is_hd || is_rg) {
                char *id = NULL, *sm = NULL;
                size_t q = p + 3;
                while (q < e) {
                    if (text[q] == '\t') { q++; continue; }
                    size_t fe = q; while (fe < e && text[fe] != '\t') fe++;
                    if (fe - q >= 3 && text[q + 2] == ':') {
                        if (is_hd && !strncmp(text + q, "SO:", 3))
                            b->so_coordinate = (fe - q - 3 == 10 && !strncmp(text + q + 3, "coordinate", 10));
                        if (is_rg && !strncmp(text + q, "ID:", 3)) { free(id); id = dupn(text + q + 3, fe - q - 3); }
                        if (is_rg && !strncmp(text + q, "SM:", 3)) { free(sm); sm = dupn(text + q + 3, fe - q - 3); }
                    }
                    q = fe;
                }
                if (is_rg) {
                    if (!id) id = dupn("", 0);
                    if (!sm) sm = dupn("", 0);
                    int sid = -1;
                    for (int i = 0; i < b->n_samples; i++) if (!strcmp(b->sample_names[i], sm)) sid = i;
                    if (sid < 0) {
                        b->sample_names = realloc(b->sample_names, (b->n_samples + 1) * sizeof(char *));
                        b->sample_names[b->n_samples] = sm; sid = b->n_samples++;
                    } else free(sm);
                    b->rg_ids = realloc(b->rg_ids, (b->n_rg + 1) * sizeof(char *));
                    b->rg_sample = realloc(b->rg_sample, (b->n_rg + 1) * sizeof(int));
                    b->rg_ids[b->n_rg] = id; b->rg_sample[b->n_rg] = sid; b->n_rg++;
                } else { free(id); free(sm); }
            }
        }
        p = e + 1;
    }
    return 0;
}

static int bam_find_ref(const Bam *b, const char *name) {
    for (int i = 0; i < b->n_ref; i++) if (!strcmp(b->refs[i].name, name)) return i;
    return -1;
}

/* ------------------------------------------------------ BAM record (layer 2)
 * record framing:  BioD/bio/std/hts/bam/readrange.d:118-173
 * fixed fields:    BioD/bio/std/hts/bam/read.d:907-972, array offsets :984-1003
 * basesCovered:    read.d:255-262     CIGAR predicates: cigar.d:58-148 (CIGAR_TYPE :116)
 * sequence[i]:     read.d:364-383     base_qualities: read.d:468-470
 * aux tag scan:    read.d:1070-1087 (linear scan, used for RG by depth.d:242)
 */
#define CIGAR_TYPE_BITS 0x3C1A7u  /* 0b11_11_00_00_01_10_10_01_11 */
static inline int op_qcons(uint32_t raw) { uint32_t s = (raw & 0xF) * 2; return s < 32 ? (CIGAR_TYPE_BITS >> s) & 1 : 0; }
static inline int op_rcons(uint32_t raw) { uint32_t s = (raw & 0xF) * 2; return s < 32 ? ((CIGAR_TYPE_BITS >> s) >> 1) & 1 : 0; }
static inline int op_match(uint32_t raw) { uint32_t s = (raw & 0xF) * 2; return s < 32 ? ((CIGAR_TYPE_BITS >> s) & 3) == 3 : 0; }
static inline uint32_t op_len(uint32_t raw) { return raw >> 4; }

typedef struct {
    const uint8_t *rec; uint32_t rec_size;   /* rec points at refID (after block_size) */
    int32_t ref_id, pos; uint32_t end_pos;
    uint16_t flag; uint8_t mapq; uint8_t l_read_name; uint16_t n_cigar; int32_t l_seq;
    const uint8_t *cigar, *seq, *qual; const char *name;
    uint64_t name_hash; uint32_t sample_id; uint8_t mate_overlap;
    /* PileupRead cursor (pileup.d:162-173) */
    uint32_t cur_op_index, cur_op, cur_op_offset, query_offset;
} PRead;

static inline uint32_t rcigar(const PRead *r, uint32_t i) { return rd32(r->cigar + 4 * (size_t)i); }

static int32_t bases_covered(const PRead *r) {
    if (r->flag & 0x4) return 0;
    int32_t n = 0;
    for (uint32_t i = 0; i < r->n_cigar; i++) { uint32_t c = rcigar(r, i); if (op_rcons(c)) n += (int32_t)op_len(c); }
    return n;
}

static const char NT16[] = "=ACMGRSVTWYHKDBN";
static const uint8_t NT16_TO_NT5[16] = {4, 0, 1, 4, 2, 4, 4, 4, 3, 4, 4, 4, 4, 4, 4, 4};  /* base.d:186 */
static inline uint8_t seq_nt16(const PRead *r, uint32_t i) { uint8_t b = r->seq[i >> 1]; return (i & 1) ? (b & 0xF) : (b >> 4); }

/* skip one aux value; returns bytes consumed or 0 on malformed */
static size_t aux_skip(const uint8_t *p, const uint8_t *end) {
    if (p >= end) return 0;
    char t = (char)*p; size_t n = 1;
    switch (t) {
    case 'A': case 'c': case 'C': n += 1; break;
    case 's': case 'S': n += 2; break;
    case 'i': case 'I': case 'f': n += 4; break;
    case 'Z': case 'H': { const uint8_t *q = p + 1; while (q < end && *q) q++; n = (size_t)(q - p) + 1; break; }
    case 'B': {
        if (p + 6 > end) return 0;
        char st = (char)p[1]; uint32_t cnt = rd32(p + 2); size_t es = (st == 'c' || st == 'C') ? 1 : (st == 's' || st == 'S') ? 2 : 4;
        n = 6 + es * cnt; break; }
    default: return 0;
    }
    return (p + n <= end) ? n : 0;
}

static int parse_record(const Bam *b, const uint8_t *rec, uint32_t rec_size, PRead *r) {
    memset(r, 0, sizeof *r);
    if (rec_size < 32) return fail("invalid BAM record (size %u)", rec_size);
    r->rec = rec; r->rec_size = rec_size;
    r->ref_id = (int32_t)rd32(rec); r->pos = (int32_t)rd32(rec + 4);
    uint32_t bmn = rd32(rec + 8), fnc = rd32(rec + 12);
    r->l_read_name = bmn & 0xFF; r->mapq = (bmn >> 8) & 0xFF;
    r->flag = (uint16_t)(fnc >> 16); r->n_cigar = (uint16_t)(fnc & 0xFFFF);
    r->l_seq = (int32_t)rd32(rec + 16);
    size_t o = 32;
    r->name = (const char *)rec + o; o += r->l_read_name;
    r->cigar = rec + o; o += 4 * (size_t)r->n_cigar;
    r->seq = rec + o; o += ((size_t)r->l_seq + 1) / 2;
    r->qual = rec + o; o += (size_t)r->l_seq;
    if (o > rec_size) return fail("invalid BAM record (fields exceed block_size)");
    r->end_pos = (uint32_t)(r->pos + bases_covered(r));   /* EagerBamRead.end_position, read.d:1378-1397 */
    /* CustomBamRead (depth.d:240-259): RG -> sample id, FNV-1a 64 of the name (without NUL) */
    uint64_t h = 14695981039346656037ULL;
    for (uint32_t i = 0; i + 1 < r->l_read_name; i++) { h ^= (uint8_t)r->name[i]; h *= 1099511628211ULL; }
    r->name_hash = h;
    r->sample_id = 0;
    if (b->n_rg > 0) {
        const uint8_t *p = rec + o, *end = rec + rec_size;
        while (p + 3 <= end) {
            if (p[0] == 'R' && p[1] == 'G' && p[2] == 'Z') {
                const char *v = (const char *)p + 3; size_t vl = strnlen(v, (size_t)(end - (p + 3)));
                int found = -1;
                for (int i = 0; i < b->n_rg; i++) if (strlen(b->rg_ids[i]) == vl && !memcmp(b->rg_ids[i], v, vl)) found = i;
                if (found < 0) return fail("error in read %s: read group %.*s is not present in the header", r->name, (int)vl, v);
                r->sample_id = (uint32_t)b->rg_sample[found];
                break;
            }
            size_t s = aux_skip(p + 2, end);
            if (!s) break;
            p += 2 + s;
        }
    }
    return 0;
}

/* PileupRead constructor, pileup.d:175-192 */
static void pread_init_cursor(PRead *r) {
    r->cur_op_index = 0; r->cur_op = 0; r->cur_op_offset = 0; r->query_offset = 0;
    for (; r->cur_op_index < r->n_cigar; ++r->cur_op_index) {
        r->cur_op = rcigar(r, r->cur_op_index);
        if (op_rcons(r->cur_op)) { if ((r->cur_op & 0xF) != 3 /* 'N' */) break; }
        else if (op_qcons(r->cur_op)) r->query_offset += op_len(r->cur_op);
    }
}
/* pileup.d:195-222 */
static void pread_increment(PRead *r) {
    ++r->cur_op_offset;
    if (op_qcons(r->cur_op)) ++r->query_offset;
    if (r->cur_op_offset >= op_len(r->cur_op)) {
        r->cur_op_offset = 0;
        for (++r->cur_op_index; r->cur_op_index < r->n_cigar; ++r->cur_op_index) {
            r->cur_op = rcigar(r, r->cur_op_index);
            if (op_rcons(r->cur_op)) break;
            if (op_qcons(r->cur_op)) r->query_offset += op_len(r->cur_op);
        }
    }
}
/* pileup.d:115-134.  '-' for D/N; out-of-range query offsets (quirk 3) read as '=' / qual 0
 * instead of the reference's unchecked memory read. */
static inline char pread_base(const PRead *r) {
    if (op_qcons(r->cur_op) && op_rcons(r->cur_op))
        return (r->query_offset < (uint32_t)r->l_seq) ? NT16[seq_nt16(r, r->query_offset)] : '=';
    return '-';
}
static inline uint8_t pread_qual(const PRead *r) {
    if (op_qcons(r->cur_op) && op_rcons(r->cur_op))
        return (r->query_offset < (uint32_t)r->l_seq) ? r->qual[r->query_offset] : 0;
    return 255;
}
static inline uint8_t base5_of_char(char c) {
    switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; }
}

/* ----------------------------------------------------------- regions / BED
 * BamRegion:   BioD/bio/std/hts/bam/region.d:28-65
 * parseBed:    sambamba/utils/common/bed.d:59-152
 * parseRegion: BioD/bio/core/region.d (region.rl:29-35): ref[:beg[-end]], 1-based closed -> 0-based half open
 */
typedef struct { uint32_t ref_id, start, end; } Region;
static int region_cmp(const void *a, const void *b) {
    const Region *x = a, *y = b;
    if (x->ref_id != y->ref_id) return x->ref_id < y->ref_id ? -1 : 1;
    if (x->start != y->start) return x->start < y->start ? -1 : 1;
    if (x->end != y->end) return x->end < y->end ? -1 : 1;
    return 0;
}
typedef struct { char *chr; long beg, end; } BedIv;
typedef struct {
    BedIv *ivs; size_t n_ivs, cap_ivs;       /* valid intervals in file order */
    char **lines; size_t n_lines, cap_lines; /* every line with >= 2 fields   */
} BedFile;

static int is_white(char c) { return c == ' ' || c == '\t' || c == '\r' || c == '\n' || c == '\v' || c == '\f'; }

/* returns 0 ok, -1 cannot read / parse (caller falls back to parseRegion, depth.d:1194) */
static int bed_read(const char *path, BedFile *bf) {
    memset(bf, 0, sizeof *bf);
    FILE *f = fopen(path, "rb"); if (!f) return -1;
    fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET);
    if (n < 0) { fclose(f); return -1; }
    char *txt = malloc(n + 1); if (fread(txt, 1, n, f) != (size_t)n) { fclose(f); free(txt); return -1; } txt[n] = 0; fclose(f);
    long p = 0;
    while (p <= n) {
        long e = p; while (e < n && txt[e] != '\n') e++;
        /* split on whitespace */
        const char *fs[3]; size_t fl[3]; int nf = 0; long q = p; int total_fields = 0;
        while (q < e) {
            while (q < e && is_white(txt[q])) q++;
            if (q >= e) break;
            long s = q; while (q < e && !is_white(txt[q])) q++;
            if (nf < 3) { fs[nf] = txt + s; fl[nf] = (size_t)(q - s); nf++; }
            total_fields++;
        }
        if (total_fields >= 2) {
            long v[2] = {0, 0};
            for (int k = 1; k < nf; k++) {
                char tmp[32]; if (fl[k] >= sizeof tmp) { free(txt); return -1; }
                memcpy(tmp, fs[k], fl[k]); tmp[fl[k]] = 0;
                char *endp; v[k - 1] = strtol(tmp, &endp, 10);
                if (*endp || endp == tmp) { free(txt); return -1; }   /* to!long throws -> fallback */
            }
            long beg = v[0], end = (nf >= 3) ? v[1] : v[0] + 1;
            if (beg == end) end = beg + 1;
            if (beg < end) { BedIv iv = { dupn(fs[0], fl[0]), beg, end }; VEC_PUSH(bf->ivs, bf->n_ivs, bf->cap_ivs, iv); }
            char *line = dupn(txt + p, (size_t)(e - p));
            VEC_PUSH(bf->lines, bf->n_lines, bf->cap_lines, line);
        }
        p = e + 1;
    }
    free(txt);
    return 0;
}

/* parseBed(non_overlapping=true): per-chromosome merge (cur.end >= next.beg merges), then sort */
static Region *bed_regions_merged(const Bam *b, const BedFile *bf, size_t *out_n) {
    Region *tmp = NULL; size_t n = 0, cap = 0;
    for (size_t i = 0; i < bf->n_ivs; i++) {
        int id = bam_find_ref(b, bf->ivs[i].chr); if (id < 0) continue;
        Region r = { (uint32_t)id, (uint32_t)bf->ivs[i].beg, (uint32_t)bf->ivs[i].end };
        VEC_PUSH(tmp, n, cap, r);
    }
    /* merge per ref on (long) begs; we merge on the uint32 casts which is identical for valid input */
    qsort(tmp, n, sizeof *tmp, region_cmp);
    size_t m = 0;
    for (size_t i = 0; i < n; i++) {
        if (m && tmp[m - 1].ref_id == tmp[i].ref_id && tmp[m - 1].end >= tmp[i].start) { if (tmp[i].end > tmp[m - 1].end) tmp[m - 1].end = tmp[i].end; }
        else tmp[m++] = tmp[i];
    }
    *out_n = m; return tmp;
}
static Region *bed_regions_raw(const Bam *b, const BedFile *bf, size_t *out_n) {
    Region *tmp = NULL; size_t n = 0, cap = 0;
    for (size_t i = 0; i < bf->n_ivs; i++) {
        int id = bam_find_ref(b, bf->ivs[i].chr); if (id < 0) continue;
        Region r = { (uint32_t)id, (uint32_t)bf->ivs[i].beg, (uint32_t)bf->ivs[i].end };
        VEC_PUSH(tmp, n, cap, r);
    }
    *out_n = n; return tmp;
}

static int parse_region_string(const char *s, char **ref, uint32_t *beg, uint32_t *end) {
    *beg = 0; *end = UINT32_MAX;
    const char *colon = strrchr(s, ':');
    /* the Ragel grammar takes the reference up to a ':' that is followed by digits/commas [- digits/commas] to the end */
    const char *c = NULL;
    for (const char *t = s; *t; t++) if (*t == ':') {
        const char *q = t + 1; int ok = (*q >= '0' && *q <= '9');
        while (*q && ((*q >= '0' && *q <= '9') || *q == ',')) q++;
        if (ok && *q == '-') { q++; if (!(*q >= '0' && *q <= '9')) ok = 0; while (*q && ((*q >= '0' && *q <= '9') || *q == ',')) q++; }
        if (ok && !*q) { c = t; break; }
    }
    (void)colon;
    if (!c) { *ref = dupn(s, strlen(s)); return 0; }
    *ref = dupn(s, (size_t)(c - s));
    long v = 0; const char *q = c + 1;
    while (*q && *q != '-') { if (*q != ',') v = v * 10 + (*q - '0'); q++; }
    *beg = (uint32_t)(v - 1);
    if (*q == '-') { q++; v = 0; while (*q) { if (*q != ',') v = v * 10 + (*q - '0'); q++; } *end = (uint32_t)v; }
    return 0;
}

/* ------------------------------------------------------------ read source
 * whole file:   BamReader.reads (reader.d:229-232)
 * with -L:      RandomAccessManager.getReads(BamRegion[]) + BamReadFilter.findNext
 *               (randomaccessmanager.d:316-338, 397-461); BAI chunk selection only
 *               narrows I/O and is not modelled.
 * filter:       depth.d:1159 default predicate; filtering.d:163-167,194-214
 * pileupColumns drops basesCovered()==0: pileup.d:509-519
 */
typedef struct {
    const Bam *b; size_t off;
    int filter_mode;            /* 0 = default, 1 = none (-F "") */
    const Region *sel; size_t n_sel, sel_idx;  /* merged sorted regions (or NULL) */
    int sel_done_ref;           /* ref whose region group is exhausted */
    int err;
} ReadSrc;

static int src_next(ReadSrc *s, PRead *out) {
    const Bgzf *z = &s->b->z;
    while (s->off + 4 <= z->ulen) {
        uint32_t bs = rd32(z->u + s->off);
        if (s->off + 4 + (size_t)bs > z->ulen) { if (z->sampled) break;   /* a bounded sample of a larger file ends where it was cut */
            fail("not enough data in stream"); s->err = 1; return 0; }   /* the stream ends inside a record: readExact throws, readrange.d:169 (fewer than 4 stray bytes end it quietly, :139-149) */
        const uint8_t *rec = z->u + s->off + 4; s->off += 4 + (size_t)bs;
        PRead r; if (parse_record(s->b, rec, bs, &r)) { s->err = 1; return 0; }
        if (s->sel) {
            /* groups are per reference in ascending ref order; within a group walk regions */
            if (r.ref_id < 0) continue;
            while (s->sel_idx < s->n_sel && s->sel[s->sel_idx].ref_id < (uint32_t)r.ref_id) s->sel_idx++;
            if (s->sel_idx >= s->n_sel) return 0;
            if (s->sel[s->sel_idx].ref_id != (uint32_t)r.ref_id) continue;
            int keep = 0;
            while (s->sel_idx < s->n_sel && s->sel[s->sel_idx].ref_id == (uint32_t)r.ref_id) {
                const Region *g = &s->sel[s->sel_idx];
                if ((uint32_t)r.pos >= g->end) { s->sel_idx++; continue; }
                if ((uint32_t)r.pos > g->start) { keep = 1; break; }
                if ((uint32_t)(r.pos + bases_covered(&r)) <= g->start) { keep = 0; break; }
                keep = 1; break;
            }
            if (!keep) continue;
        }
        if (s->filter_mode == 0) { if (!(r.mapq > 0) || (r.flag & 0x400) || (r.flag & 0x200)) continue; }
        if (bases_covered(&r) <= 0) continue;
        *out = r; return 1;
    }
    return 0;
}

/* ------------------------------------------------------------ column sweep
 * PileupRange.popFront / initNewReference: pileup.d:345-424 (skip_zero_coverage = true)
 */
typedef struct {
    ReadSrc *src; PRead look; int has_look;
    PRead *reads; size_t n, cap;
    int ref_id; uint64_t position; size_t n_starting_here;
    int started;
} Sweep;

static void sweep_add(Sweep *w, const PRead *r) { PRead t = *r; pread_init_cursor(&t); VEC_PUSH(w->reads, w->n, w->cap, t); }
static void sweep_pull(Sweep *w) { w->has_look = src_next(w->src, &w->look); }
static void sweep_init_new_reference(Sweep *w) {
    w->position = (uint64_t)(uint32_t)w->look.pos; w->ref_id = w->look.ref_id;
    size_t n = 1; sweep_add(w, &w->look); sweep_pull(w);
    while (w->has_look && w->look.ref_id == w->ref_id && (uint64_t)(uint32_t)w->look.pos == w->position) { sweep_add(w, &w->look); n++; sweep_pull(w); }
    w->n_starting_here = n;
}
static int sweep_empty(const Sweep *w) { return !w->has_look && w->n == 0; }
static void sweep_start(Sweep *w, ReadSrc *src) { memset(w, 0, sizeof *w); w->src = src; w->ref_id = -1; sweep_pull(w); if (w->has_look) sweep_init_new_reference(w); }
static void sweep_pop(Sweep *w) {
    uint64_t pos = ++w->position; size_t survived = 0;
    for (size_t i = 0; i < w->n; i++) if ((uint64_t)w->reads[i].end_pos > pos) { if (survived < i) w->reads[survived] = w->reads[i]; survived++; }
    for (size_t i = 0; i < survived; i++) pread_increment(&w->reads[i]);
    w->n = survived; w->n_starting_here = 0;
    if (w->has_look) {
        if (w->look.ref_id != w->ref_id && survived == 0) sweep_init_new_reference(w);
        else {
            size_t n = 0;
            while (w->has_look && (uint64_t)(uint32_t)w->look.pos == pos && w->look.ref_id == w->ref_id) { sweep_add(w, &w->look); sweep_pull(w); n++; }
            w->n_starting_here = n;
            if (survived == 0 && n == 0) sweep_init_new_reference(w);
        }
    }
}

/* ------------------------------------------------------------ printer state
 * ColumnPrinter: depth.d:277-400
 */
enum { MO_NONE = 0, MO_DETECTED = 1, MO_FIXED = 2, MO_PAST = 3 };
typedef struct { uint64_t h; size_t idx; } HashIdx;
typedef struct { size_t a, b; } Pair;

typedef struct {
    int mode;                         /* 0 base, 1 region, 2 window */
    double min_cov, max_cov; int min_bq; int combined, annotate, fix_mates;
    FILE *out; const Bam *bam;
    int n_samples; char **sample_names;
    /* mates */
    HashIdx *hbuf; size_t hcap; Pair *pairs; size_t n_pairs, pcap;
    /* base */
    int report_zero; int prev_ref_id; long prev_position; int bed_provided;
    Region *bed; size_t n_bed, bed_front;          /* merged regions, mutable front (base -L) */
    size_t col_idx;                                 /* NonOverlappingRegionStatsCollector cursor */
    /* region / window */
    Region *raw_bed; size_t n_raw_bed; char **raw_bed_lines; size_t n_raw_lines;
    int general_collector; size_t nonov_idx;
    uint32_t *thr; size_t n_thr;
    uint32_t **cov_cnt; /* [sample][thr*n_regions] */ uint32_t **n_reads, **n_bases; size_t n_regions;
    uint8_t *first_occ; uint32_t *cov_per_sample; int n_sdata;
    size_t window_size, overlap, step, nwin, leftmost_index, leftmost_start; int window_ref_id; size_t ref_length;
} Printer;

static uint32_t sample_of(const Printer *p, const PRead *r) { return (p->combined || p->n_samples == 1) ? 0 : r->sample_id; }

static int hcmp(const void *a, const void *b) { const HashIdx *x = a, *y = b; if (x->h != y->h) return x->h < y->h ? -1 : 1; return x->idx < y->idx ? -1 : (x->idx > y->idx); }

/* depth.d:319-388.  D's sort is unstable; ties (equal hashes) are exactly the mate pairs, whose
 * treatment is symmetric except for selectBetterMate's tie-break, so we order ties by index. */
static void detect_overlapping_mates(Printer *p, Sweep *w) {
    p->n_pairs = 0;
    if (!p->fix_mates) return;
    size_t n = w->n; if (n == 0) return;
    if (n > p->hcap) { p->hcap = n * 2; p->hbuf = realloc(p->hbuf, p->hcap * sizeof *p->hbuf); }
    for (size_t i = 0; i < n; i++) { p->hbuf[i].h = w->reads[i].name_hash; p->hbuf[i].idx = i; }
    qsort(p->hbuf, n, sizeof *p->hbuf, hcmp);
    for (size_t i = 0; i + 1 < n; i++) {
        if (p->hbuf[i].h != p->hbuf[i + 1].h) {
            size_t idx = p->hbuf[i].idx;
            if (w->reads[idx].mate_overlap != MO_NONE) w->reads[idx].mate_overlap = MO_PAST;
            continue;
        }
        size_t i1 = p->hbuf[i].idx, i2 = p->hbuf[i + 1].idx; PRead *r1 = &w->reads[i1], *r2 = &w->reads[i2];
        if (r1->sample_id == r2->sample_id && r1->l_read_name == r2->l_read_name && !memcmp(r1->name, r2->name, r1->l_read_name)) {
            if (r1->mate_overlap != MO_NONE && r2->mate_overlap != MO_NONE && r1->mate_overlap == r2->mate_overlap)
                fprintf(stderr, "[WARNING] mates overlap in index %d\n", (int)r1->mate_overlap);
            Pair pr = { i1, i2 }; VEC_PUSH(p->pairs, p->n_pairs, p->pcap, pr);
            if (r1->mate_overlap == MO_NONE) r1->mate_overlap = MO_DETECTED;
            if (r2->mate_overlap == MO_NONE) r2->mate_overlap = MO_DETECTED;
            i += 1;
        }
    }
    size_t idx = p->hbuf[n - 1].idx;
    if (w->reads[idx].mate_overlap != MO_NONE && (n == 1 || p->hbuf[n - 2].h != p->hbuf[n - 1].h)) w->reads[idx].mate_overlap = MO_PAST;
}
/* depth.d:391-399 */
static PRead *select_better_mate(PRead *m1, PRead *m2) {
    if (pread_base(m1) == '-' || pread_base(m2) == '-') return m1->mapq > m2->mapq ? m1 : m2;
    return pread_qual(m1) > pread_qual(m2) ? m1 : m2;
}

/* -------------------------------------------------------------- base mode
 * PerBasePrinter: depth.d:402-607
 */
static void base_header(Printer *p) {
    fputs("REF\tPOS\tCOV\tA\tC\tG\tT\tDEL\tREFSKIP", p->out);
    if (!p->combined) fputs("\tSAMPLE", p->out);
    if (p->annotate) fputs("\tFLAG", p->out);
    fputc('\n', p->out);
}
static void base_write_tail_rows(Printer *p, const char *ref_name, long pos) {
    int ns = p->combined ? 1 : p->n_samples;
    for (int s = 0; s < ns; s++) {
        fprintf(p->out, "%s\t%ld\t0\t0\t0\t0\t0\t0\t0", ref_name, pos);
        if (!p->combined) fprintf(p->out, "\t%s", p->sample_names[s]);
        if (p->annotate) fputs(p->min_cov > 0 ? "\tn" : "\ty", p->out);
        fputc('\n', p->out);
    }
}
static int region_fully_left(const Region *r, uint32_t ref_id, uint32_t pos) { return r->ref_id < ref_id || (r->ref_id == ref_id && r->end <= pos); }
static int region_overlaps(const Region *r, uint32_t ref_id, uint32_t pos) { return r->ref_id == ref_id && r->start <= pos && pos < r->end; }

static void base_write_empty(Printer *p, long ref_id, long start, long end) {     /* depth.d:452-487 */
    if (p->min_cov > 0 && !p->annotate) return;
    const char *ref_name = p->bam->refs[(uint32_t)ref_id].name;
    if (!p->bed_provided) { for (long pos = start; pos < end; pos++) base_write_tail_rows(p, ref_name, pos); return; }
    if (p->bed_front >= p->n_bed || p->bed[p->bed_front].ref_id > (uint32_t)ref_id) return;
    while (p->bed_front < p->n_bed && p->bed[p->bed_front].ref_id < (uint32_t)ref_id) p->bed_front++;
    while (p->bed_front < p->n_bed && p->bed[p->bed_front].ref_id == (uint32_t)ref_id) {
        Region *g = &p->bed[p->bed_front];
        if (region_fully_left(g, (uint32_t)ref_id, (uint32_t)start)) { p->bed_front++; continue; }
        long from = start > (long)g->start ? start : (long)g->start, to = end < (long)g->end ? end : (long)g->end;
        if (from >= to) break;
        for (long pos = from; pos < to; pos++) base_write_tail_rows(p, ref_name, pos);
        g->start = (uint32_t)to;
        if (g->start >= g->end) p->bed_front++;
    }
    p->col_idx = p->bed_front;   /* stats_collector rebuilt over the remaining raw_bed */
}
static int base_output_required(Printer *p, int ref_id, uint64_t position) {        /* depth.d:558-565, 182-197 */
    if (!p->bed_provided) return 1;
    while (p->col_idx < p->n_bed && region_fully_left(&p->bed[p->col_idx], (uint32_t)ref_id, (uint32_t)position)) p->col_idx++;
    return p->col_idx < p->n_bed && region_overlaps(&p->bed[p->col_idx], (uint32_t)ref_id, (uint32_t)position);
}
static void base_process_current(Printer *p, const PRead *r, size_t *cov, size_t *del, size_t *skip) {
    uint32_t s = sample_of(p, r);
    char c = pread_base(r);
    if (c == '-') { if ((r->cur_op & 0xF) == 2) del[s]++; else skip[s]++; return; }
    if (pread_qual(r) >= p->min_bq) cov[5 * s + base5_of_char(c)]++;
}
static void base_write_column(Printer *p, Sweep *w) {                                 /* depth.d:495-556 */
    int ns = p->combined ? 1 : p->n_samples; if (ns < 1) ns = 1;
    size_t cov[5 * 64] = {0}, del[64] = {0}, skip[64] = {0};
    size_t *covp = cov, *delp = del, *skipp = skip;
    if (ns > 64) { covp = calloc(5 * ns, sizeof *covp); delp = calloc(ns, sizeof *delp); skipp = calloc(ns, sizeof *skipp); }
    detect_overlapping_mates(p, w);
    for (size_t i = 0; i < w->n; i++) { if (w->reads[i].mate_overlap == MO_DETECTED) continue; base_process_current(p, &w->reads[i], covp, delp, skipp); }
    for (size_t k = 0; k < p->n_pairs; k++) base_process_current(p, select_better_mate(&w->reads[p->pairs[k].a], &w->reads[p->pairs[k].b]), covp, delp, skipp);
    for (int s = 0; s < ns; s++) {
        size_t total = covp[5 * s] + covp[5 * s + 1] + covp[5 * s + 2] + covp[5 * s + 3] + covp[5 * s + 4] + delp[s] + skipp[s];
        int ok = (double)total >= p->min_cov && (double)total <= p->max_cov;
        if (!ok && !p->annotate) break;          /* `return`, not `continue` (quirk 2) */
        fprintf(p->out, "%s\t%llu\t%zu\t%zu\t%zu\t%zu\t%zu\t%zu\t%zu", p->bam->refs[w->ref_id].name, (unsigned long long)w->position, total,
                covp[5 * s], covp[5 * s + 1], covp[5 * s + 2], covp[5 * s + 3], delp[s], skipp[s]);
        if (!p->combined) fprintf(p->out, "\t%s", p->sample_names[s]);
        if (p->annotate) fputs(ok ? "\ty" : "\tn", p->out);
        fputc('\n', p->out);
    }
    if (ns > 64) { free(covp); free(delp); free(skipp); }
}
static void base_push(Printer *p, Sweep *w) {                                         /* depth.d:567-591 */
    if (p->min_cov > 0) { if (base_output_required(p, w->ref_id, w->position)) base_write_column(p, w); return; }
    if (p->prev_ref_id == -2) {
        for (int id = 0; id < w->ref_id; id++) base_write_empty(p, id, 0, p->bam->refs[id].length);
        base_write_empty(p, w->ref_id, 0, (long)w->position);
    } else if (p->prev_ref_id != w->ref_id) {
        base_write_empty(p, p->prev_ref_id, p->prev_position + 1, p->bam->refs[p->prev_ref_id].length);
        base_write_empty(p, w->ref_id, 0, (long)w->position);
    } else if (p->prev_position != (long)w->position - 1) base_write_empty(p, w->ref_id, p->prev_position + 1, (long)w->position);
    p->prev_ref_id = w->ref_id; p->prev_position = (long)w->position;
    if (base_output_required(p, w->ref_id, w->position)) base_write_column(p, w);
}
static void base_close(Printer *p) {                                                  /* depth.d:593-606 */
    if (!p->report_zero) return;
    if (p->prev_ref_id == -2) { for (int id = 0; id < p->bam->n_ref; id++) base_write_empty(p, id, 0, p->bam->refs[id].length); }
    else {
        base_write_empty(p, p->prev_ref_id, p->prev_position + 1, p->bam->refs[p->prev_ref_id].length);
        for (int id = p->prev_ref_id + 1; id < p->bam->n_ref; id++) base_write_empty(p, id, 0, p->bam->refs[id].length);
    }
}

/* ------------------------------------------------- region and window modes
 * PerRegionPrinter: depth.d:637-877; PerBedRegionPrinter :879-931; PerWindowPrinter :933-1077
 * collectors: depth.d:112-227
 */
static void fmt_float(FILE *f, float v) { fprintf(f, "%g", (double)v); }   /* D write(float) == %g, 6 significant digits */

static void region_alloc(Printer *p, size_t n_regions) {
    p->n_regions = n_regions; p->n_sdata = p->combined ? 1 : p->n_samples; if (p->n_sdata < 1) p->n_sdata = 1;
    p->cov_cnt = calloc(p->n_sdata, sizeof *p->cov_cnt); p->n_reads = calloc(p->n_sdata, sizeof *p->n_reads); p->n_bases = calloc(p->n_sdata, sizeof *p->n_bases);
    for (int s = 0; s < p->n_sdata; s++) {
        p->cov_cnt[s] = calloc((p->n_thr ? p->n_thr : 1) * (n_regions ? n_regions : 1), sizeof(uint32_t));
        p->n_reads[s] = calloc(n_regions ? n_regions : 1, sizeof(uint32_t)); p->n_bases[s] = calloc(n_regions ? n_regions : 1, sizeof(uint32_t));
    }
    p->cov_per_sample = calloc(p->n_sdata, sizeof(uint32_t));
    p->first_occ = malloc(n_regions ? n_regions : 1);
}
static void region_print_header(Printer *p, size_t n_before) {                       /* depth.d:643-659 */
    static const char *def[3] = {"chrom", "chromStart", "chromEnd"};
    fputs("# ", p->out);
    for (size_t k = 0; k < (n_before < 3 ? n_before : 3); k++) fprintf(p->out, "%s\t", def[k]);
    for (size_t k = 3; k < n_before; k++) fprintf(p->out, "F%zu\t", k);
    fputs("readCount\tmeanCoverage", p->out);
    for (size_t k = 0; k < p->n_thr; k++) fprintf(p->out, "\tpercentage%u", p->thr[k]);
    if (!p->combined) fputs("\tsampleName", p->out);
    if (p->annotate) fputs("\tmeanCovWithinBounds", p->out);
    fputc('\n', p->out); fflush(p->out);
}
static size_t window_start_of(const Printer *p, size_t id) {                          /* depth.d:974-982 */
    size_t k = id >= p->leftmost_index ? id - p->leftmost_index : p->nwin - p->leftmost_index + id;
    return p->leftmost_start + p->step * k;
}
static Region region_by_id(const Printer *p, size_t id) {
    if (p->mode == 1) return p->raw_bed[id];
    size_t s = window_start_of(p, id); Region r = { (uint32_t)p->window_ref_id, (uint32_t)s, (uint32_t)(s + p->window_size) }; return r;
}
static size_t count_overlapping_bases(const Printer *p, const PRead *r, size_t id, uint64_t start_pos) {   /* depth.d:671-698 */
    Region g = region_by_id(p, id);
    uint32_t pos = (uint32_t)r->pos; size_t n = 0; uint32_t q = 0, lq = (uint32_t)(r->l_seq > 0 ? r->l_seq : 0);
    for (uint32_t i = 0; i < r->n_cigar; i++) {
        uint32_t c = rcigar(r, i), len = op_len(c);
        uint32_t avail = q < lq ? lq - q : 0, m = len < avail ? len : avail;
        if (op_match(c)) { for (uint32_t k = 0; k < m; k++) { n += (g.start <= pos && pos < g.end) && r->qual[q + k] >= p->min_bq && pos >= start_pos; ++pos; } }
        else if (op_rcons(c)) pos += len;
        if (op_qcons(c)) q += m;
    }
    return n;
}
static void count_read(Printer *p, const PRead *r, size_t id) {                        /* depth.d:661-669 */
    size_t n = count_overlapping_bases(p, r, id, 0); uint32_t s = sample_of(p, r);
    p->n_bases[s][id] += (uint32_t)n; if (n > 0) p->n_reads[s][id] += 1;
}
static void uncount_overlapping_mates(Printer *p, PRead *r1, PRead *r2, size_t id, uint64_t curr_pos) {    /* depth.d:717-743 */
    if (r1->mate_overlap == MO_FIXED && r2->mate_overlap == MO_FIXED) return;
    size_t n1f = count_overlapping_bases(p, r1, id, 0), n2f = count_overlapping_bases(p, r2, id, 0);
    size_t n1 = (uint64_t)(uint32_t)r1->pos == curr_pos ? n1f : count_overlapping_bases(p, r1, id, curr_pos);
    size_t n2 = (uint64_t)(uint32_t)r2->pos == curr_pos ? n2f : count_overlapping_bases(p, r2, id, curr_pos);
    uint32_t s = r1->sample_id; if (s >= (uint32_t)p->n_sdata) s = 0;   /* reference indexes samples[r1.sample_id] directly */
    p->n_bases[s][id] -= (uint32_t)(n1 + n2);
    p->n_reads[s][id] -= (uint32_t)((n1f > 0) + (n2f > 0));
    p->n_reads[s][id] += (uint32_t)(n1f + n2f > 0);
}
static void region_update(Printer *p, Sweep *w, size_t id, int *fixes_applied) {       /* body of the delegate, depth.d:801-841 */
    if (p->first_occ[id]) {
        for (size_t i = 0; i < w->n; i++) if (w->reads[i].mate_overlap != MO_FIXED) count_read(p, &w->reads[i], id);
        for (size_t k = 0; k < p->n_pairs; k++) {           /* countPreviouslySeenMateOverlaps */
            PRead *m1 = &w->reads[p->pairs[k].a], *m2 = &w->reads[p->pairs[k].b];
            if (m1->mate_overlap != MO_FIXED) continue;
            size_t n1 = count_overlapping_bases(p, m1, id, 0), n2 = count_overlapping_bases(p, m2, id, 0);
            if (n1 + n2 == 0) continue;
            uint32_t s = m1->sample_id; if (s >= (uint32_t)p->n_sdata) s = 0;
            p->n_reads[s][id] += 1;
        }
        p->first_occ[id] = 0;
    } else {
        for (size_t i = w->n - w->n_starting_here; i < w->n; i++) count_read(p, &w->reads[i], id);
    }
    for (size_t k = 0; k < p->n_pairs; k++) uncount_overlapping_mates(p, &w->reads[p->pairs[k].a], &w->reads[p->pairs[k].b], id, w->position);
    *fixes_applied = 1;
    memset(p->cov_per_sample, 0, p->n_sdata * sizeof(uint32_t));
    for (size_t i = 0; i < w->n; i++) {
        PRead *r = &w->reads[i];
        if (r->mate_overlap != MO_NONE) {
            if (r->mate_overlap != MO_PAST) continue;
            if (pread_qual(r) < p->min_bq) continue;
            uint32_t s = sample_of(p, r); p->n_bases[s][id] += 1; p->cov_per_sample[s] += 1;
        } else if (pread_qual(r) >= p->min_bq) p->cov_per_sample[sample_of(p, r)] += 1;
    }
    for (size_t k = 0; k < p->n_pairs; k++) {
        PRead *r = select_better_mate(&w->reads[p->pairs[k].a], &w->reads[p->pairs[k].b]);
        if (pread_qual(r) < p->min_bq) continue;
        uint32_t s = sample_of(p, r); p->n_bases[s][id] += 1; p->cov_per_sample[s] += 1;
    }
    for (int s = 0; s < p->n_sdata; s++) for (size_t t = 0; t < p->n_thr; t++) if (p->cov_per_sample[s] >= p->thr[t]) p->cov_cnt[s][t * p->n_regions + id] += 1;
}
static void region_push(Printer *p, Sweep *w) {                                         /* depth.d:760-845 */
    uint32_t ref_id = (uint32_t)w->ref_id, position = (uint32_t)w->position;
    detect_overlapping_mates(p, w);
    int fixes_applied = 0;
    if (p->mode == 2) {                                  /* WindowStatsCollector.nextColumn, depth.d:215-226 */
        size_t k = position < p->window_size ? position / p->step + 1 : p->nwin;
        for (size_t id = 0; id < k; id++) region_update(p, w, id, &fixes_applied);
    } else if (!p->general_collector) {                  /* NonOverlappingRegionStatsCollector, depth.d:182-197 */
        while (p->nonov_idx < p->n_raw_bed && region_fully_left(&p->raw_bed[p->nonov_idx], ref_id, position)) p->nonov_idx++;
        if (p->nonov_idx < p->n_raw_bed && region_overlaps(&p->raw_bed[p->nonov_idx], ref_id, position)) region_update(p, w, p->nonov_idx, &fixes_applied);
    } else {                                             /* GeneralRegionStatsCollector (interval tree), depth.d:143-152 */
        for (size_t id = 0; id < p->n_raw_bed; id++) if (region_overlaps(&p->raw_bed[id], ref_id, position)) region_update(p, w, id, &fixes_applied);
    }
    if (fixes_applied) for (size_t k = 0; k < p->n_pairs; k++) { w->reads[p->pairs[k].a].mate_overlap = MO_FIXED; w->reads[p->pairs[k].b].mate_overlap = MO_FIXED; }
}
static void region_print_stats(Printer *p, int s, size_t id) {                           /* depth.d:847-876 */
    Region g = region_by_id(p, id); uint32_t length = g.end - g.start;
    float mean_cov = (float)p->n_bases[s][id] / (float)length;
    int ok = (double)mean_cov >= p->min_cov && (double)mean_cov <= p->max_cov;
    if (!ok && !p->annotate) return;
    if (p->mode == 1) {                                   /* writeOriginalBedLine, depth.d:902-906 (stripRight) */
        char *l = p->raw_bed_lines[id]; size_t n = strlen(l); while (n && is_white(l[n - 1])) l[--n] = 0;
        fprintf(p->out, "%s\t", l);
    } else fprintf(p->out, "%s\t%u\t%u\t", p->bam->refs[g.ref_id].name, g.start, g.end);
    fprintf(p->out, "%u\t", p->n_reads[s][id]); fmt_float(p->out, mean_cov);
    for (size_t j = 0; j < p->n_thr; j++) {
        float pct = (float)p->cov_cnt[s][j * p->n_regions + id] * 100 / (float)length;
        if (p->thr[j] == 0) pct = 100.0f;
        fputc('\t', p->out); fmt_float(p->out, pct);
    }
    if (!p->combined) fprintf(p->out, "\t%s", p->sample_names[s]);
    if (p->annotate) fputs(ok ? "\ty" : "\tn", p->out);
    fputc('\n', p->out); fflush(p->out);
}
static void window_reset_slot(Printer *p, size_t id) { for (int s = 0; s < p->n_sdata; s++) { p->n_reads[s][id] = 0; p->n_bases[s][id] = 0; for (size_t t = 0; t < p->n_thr; t++) p->cov_cnt[s][t * p->n_regions + id] = 0; } }
static void window_finish_leftmost(Printer *p) {                                         /* depth.d:962-972 */
    for (int s = 0; s < p->n_sdata; s++) region_print_stats(p, s, p->leftmost_index);
    window_reset_slot(p, p->leftmost_index); p->first_occ[p->leftmost_index] = 1;
    if (++p->leftmost_index == p->nwin) p->leftmost_index = 0;
    p->leftmost_start += p->step;
}
static void window_reset_all(Printer *p) { for (size_t id = 0; id < p->nwin; id++) { window_reset_slot(p, id); p->first_occ[id] = 1; } p->leftmost_index = 0; p->leftmost_start = 0; }
static void window_print_empty(Printer *p, int ref_id) {                                 /* depth.d:1039-1044 */
    p->window_ref_id = ref_id;
    size_t cnt = p->bam->refs[ref_id].length / p->step;
    for (size_t j = 0; j < cnt; j++) window_finish_leftmost(p);
    window_reset_all(p);
}
static void window_push(Printer *p, Sweep *w) {                                          /* depth.d:1051-1068 */
    if (p->window_ref_id == -1) {
        for (int k = 0; k < w->ref_id; k++) window_print_empty(p, k);
        p->window_ref_id = w->ref_id; p->ref_length = p->bam->refs[w->ref_id].length;
    } else if (w->ref_id != p->window_ref_id) {
        while (p->leftmost_start + p->window_size <= p->ref_length) window_finish_leftmost(p);
        window_reset_all(p);
        for (int k = p->window_ref_id + 1; k < w->ref_id; k++) window_print_empty(p, k);
        p->window_ref_id = w->ref_id; p->ref_length = p->bam->refs[w->ref_id].length;
    }
    while (w->position >= p->leftmost_start + p->window_size) window_finish_leftmost(p);
    region_push(p, w);
}
static void window_close(Printer *p) {                                                   /* depth.d:1070-1076 */
    while (p->leftmost_start + p->window_size <= p->ref_length) window_finish_leftmost(p);
    for (int k = p->window_ref_id + 1; k < p->bam->n_ref; k++) window_print_empty(p, k);
}

/* ------------------------------------------------------------- depth_main
 * sambamba/depth.d:1079-1245.  Option grammar: std.getopt, caseSensitive, passThrough; bundling off.
 */
static void usage(void) {
    fputs("Usage: sambamba-depth region|window|base [options] input.bam  [input2.bam [...]]\n", stderr);
}
typedef struct { int argc; char **argv; } Args;
/* fetch "-x VAL", "-xVAL", "--long VAL", "--long=VAL"; removes consumed args. Returns #found (last wins) or -1 */
static int opt_take(Args *a, const char *lng, char sht, int has_val, const char **val, int multi, void (*cb)(const char *, void *), void *ud) {
    int found = 0;
    for (int i = 1; i < a->argc; ) {
        char *s = a->argv[i]; int consumed = 0; const char *v = NULL;
        if (!strcmp(s, "--")) break;
        if (s[0] == '-' && s[1] == '-' && lng) {
            size_t ln = strlen(lng);
            if (!strncmp(s + 2, lng, ln) && (s[2 + ln] == 0 || s[2 + ln] == '=')) {
                if (!has_val) { if (s[2 + ln] == 0) consumed = 1; }
                else if (s[2 + ln] == '=') { v = s + 3 + ln; consumed = 1; }
                else if (i + 1 < a->argc) { v = a->argv[i + 1]; consumed = 2; }
                else return -1;
            }
        } else if (s[0] == '-' && s[1] != '-' && sht && s[1] == sht) {
            if (!has_val) { if (s[2] == 0) consumed = 1; }
            else if (s[2] == '=') { v = s + 3; consumed = 1; }
            else if (s[2]) { v = s + 2; consumed = 1; }
            else if (i + 1 < a->argc) { v = a->argv[i + 1]; consumed = 2; }
            else return -1;
        }
        if (consumed) {
            found++;
            if (has_val) { if (multi && cb) cb(v, ud); else if (val) *val = v; }
            memmove(&a->argv[i], &a->argv[i + consumed], (a->argc - i - consumed) * sizeof(char *)); a->argc -= consumed;
        } else i++;
    }
    return found;
}
/* std.getopt converts option values with std.conv.to!T; its exceptions end depth_main with "sambamba-depth: <message>", exit code 1
 * (depth.d:1236-1243).  Unsigned types: digits only (no sign), overflow is an error; double: what strtod consumes entirely. */
static const char *g_conv_err = NULL; static char g_conv_buf[160];
static int conv_unsigned(const char *s, unsigned long long maxv, const char *type, unsigned long long *out) {
    if (!s || !*s) { snprintf(g_conv_buf, sizeof g_conv_buf, "Unexpected end of input when converting from type string to type %s", type); g_conv_err = g_conv_buf; return 0; }
    unsigned long long v = 0;
    for (const char *c = s; *c; c++) {
        if (*c < '0' || *c > '9') { snprintf(g_conv_buf, sizeof g_conv_buf, "Unexpected '%c' when converting from type string to type %s", *c, type); g_conv_err = g_conv_buf; return 0; }
        if (v > (maxv - (unsigned)(*c - '0')) / 10) { g_conv_err = "Conversion positive overflow"; return 0; }
        v = v * 10 + (unsigned)(*c - '0');
    }
    *out = v; return 1;
}
static int conv_double(const char *s, double *out) {
    char *end = NULL; if (!s || !*s || *s == ' ' || *s == '\t') { g_conv_err = "no digits seen"; return 0; }
    double v = strtod(s, &end); if (end == s || *end) { g_conv_err = "no digits seen"; return 0; }
    *out = v; return 1;
}
static void thr_cb(const char *v, void *ud) { Printer *p = ud; unsigned long long u = 0; if (!conv_unsigned(v, 0xFFFFFFFFull, "uint", &u)) return; p->thr = realloc(p->thr, (p->n_thr + 1) * sizeof(uint32_t)); p->thr[p->n_thr++] = (uint32_t)u; }

typedef struct { int nthreads; size_t max_file_bytes; double t_inflate, t_sweep; uint64_t columns; uint64_t file_bytes; } RunStats;
static RunStats g_stats;
static double now_s(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec + ts.tv_nsec * 1e-9; }

int oracle_depth_main(int argc, char **argv_in, FILE *out_default, int inflate_threads, size_t max_file_bytes) {
    if (argc < 3) { usage(); return 0; }
    char **argv = malloc((argc + 1) * sizeof(char *)); memcpy(argv, argv_in, argc * sizeof(char *)); argv[argc] = NULL;
    Printer P; memset(&P, 0, sizeof P); P.max_cov = 1e50; P.prev_ref_id = -2; P.window_ref_id = -1;
    if (!strcmp(argv[1], "base")) P.mode = 0; else if (!strcmp(argv[1], "region")) P.mode = 1; else if (!strcmp(argv[1], "window")) P.mode = 2; else { usage(); free(argv); return 0; }
    if (P.mode == 0) P.min_cov = 1;
    Args a = { argc - 1, argv + 1 };
    const char *query = NULL, *out_fn = NULL, *v = NULL, *bed_fn = NULL; int rc = 1;
    Bam B; memset(&B, 0, sizeof B); BedFile bf; memset(&bf, 0, sizeof bf);
    FILE *out = NULL;
#define BAIL(...) do { fail(__VA_ARGS__); goto error; } while (0)
    if (opt_take(&a, "filter", 'F', 1, &query, 0, NULL, NULL) < 0) BAIL("Missing value for argument -F.");
    opt_take(&a, "output-filename", 'o', 1, &out_fn, 0, NULL, NULL);
    v = NULL; if (opt_take(&a, "nthreads", 't', 1, &v, 0, NULL, NULL) > 0 && v && inflate_threads <= 0) inflate_threads = atoi(v);
    unsigned long long uv = 0; g_conv_err = NULL;
    v = NULL; if (opt_take(&a, "min-coverage", 'c', 1, &v, 0, NULL, NULL) > 0 && !conv_double(v, &P.min_cov)) BAIL("%s", g_conv_err);
    v = NULL; if (opt_take(&a, "max-coverage", 'C', 1, &v, 0, NULL, NULL) > 0 && !conv_double(v, &P.max_cov)) BAIL("%s", g_conv_err);
    v = NULL; if (opt_take(&a, "min-base-quality", 'q', 1, &v, 0, NULL, NULL) > 0) { if (!conv_unsigned(v, 255, "ubyte", &uv)) BAIL("%s", g_conv_err); P.min_bq = (int)uv; }      /* ubyte min_base_quality, depth.d:280 */
    if (opt_take(&a, "annotate", 'a', 0, NULL, 0, NULL, NULL) > 0) P.annotate = 1;
    if (opt_take(&a, "combined", 0, 0, NULL, 0, NULL, NULL) > 0) P.combined = 1;
    if (opt_take(&a, "fix-mate-overlaps", 'm', 0, NULL, 0, NULL, NULL) > 0) P.fix_mates = 1;
    out = out_fn ? fopen(out_fn, "w+") : out_default;
    if (!out) BAIL("Cannot open file `%s' in mode `w+'", out_fn);
    { static char obuf[1 << 20]; if (out_fn) setvbuf(out, obuf, _IOFBF, sizeof obuf); }
    P.out = out;
    if (P.mode != 2) opt_take(&a, "regions", 'L', 1, &bed_fn, 0, NULL, NULL);
    if (P.mode == 1 && !bed_fn) { fputs("BED file or a region must be provided in region mode\n", stderr); free(argv); return 1; }

    /* printer.init(args): per-mode options and header line */
    if (P.mode == 0) {
        if (opt_take(&a, "report-zero-coverage", 'z', 0, NULL, 0, NULL, NULL) > 0) P.report_zero = 1;
        if (P.report_zero) P.min_cov = 0;
        if (P.min_cov == 0) P.report_zero = 1;
    } else if (P.mode == 1) {
        opt_take(&a, "cov-threshold", 'T', 1, NULL, 1, thr_cb, &P); if (g_conv_err) BAIL("%s", g_conv_err);
    } else {
        v = NULL; if (opt_take(&a, "window-size", 'w', 1, &v, 0, NULL, NULL) > 0) { if (!conv_unsigned(v, 0xFFFFFFFFFFFFFFF0ull, "ulong", &uv)) BAIL("%s", g_conv_err); P.window_size = uv; }
        v = NULL; if (opt_take(&a, "overlap", 0, 1, &v, 0, NULL, NULL) > 0) { if (!conv_unsigned(v, 0xFFFFFFFFFFFFFFF0ull, "ulong", &uv)) BAIL("%s", g_conv_err); P.overlap = uv; }
        opt_take(&a, "cov-threshold", 'T', 1, NULL, 1, thr_cb, &P); if (g_conv_err) BAIL("%s", g_conv_err);
    }
    if (a.argc < 2) BAIL("no input BAM given");
    if (a.argc > 2) BAIL("oracle supports a single BAM file");   /* multi-BAM merge is out of scope (SURVEY 2) */
    const char *bam_path = a.argv[1];

    /* base/window headers are printed by init() BEFORE the BAM is opened (depth.d:1152 then :1163) */
    if (P.mode == 0) base_header(&P);
    if (P.mode == 2) {
        if (!(P.window_size > 0)) BAIL("positive window size must be specified");
        if (!(P.overlap < P.window_size)) BAIL("specified overlap is larger than window size");
        P.step = P.window_size - P.overlap; P.nwin = P.window_size / P.step; if (P.window_size % P.step) P.nwin++;
    }
    int filter_mode = 0;
    if (query) {
        if (!*query) filter_mode = 1;
        else if (!strcmp(query, "mapping_quality > 0 and not duplicate and not failed_quality_control")) filter_mode = 0;
        else BAIL("oracle supports only the default filter or -F \"\"");
    }

    double t0 = now_s();
    if (bgzf_load(&B.z, bam_path, inflate_threads, max_file_bytes)) goto error;
    g_stats.t_inflate = now_s() - t0; g_stats.file_bytes = B.z.file_len;
    if (bam_parse_header(&B, max_file_bytes != 0)) goto error;
    if (!B.so_coordinate) BAIL("All files must be coordinate-sorted");
    {   /* has_index: <file>.bai or <file minus .bam>.bai must exist (BioD reader.d has_index) */
        char path[4096]; snprintf(path, sizeof path, "%s.bai", bam_path); FILE *f = fopen(path, "rb");
        if (!f) { size_t n = strlen(bam_path); if (n > 4 && !strcmp(bam_path + n - 4, ".bam")) { snprintf(path, sizeof path, "%.*s.bai", (int)(n - 4), bam_path); f = fopen(path, "rb"); } }
        if (!f) BAIL("All files must be indexed"); fclose(f);
    }
    P.bam = &B;
    if (B.n_samples == 0) { static char *star[] = { "*" }; P.n_samples = 1; P.sample_names = star; } else { P.n_samples = B.n_samples; P.sample_names = B.sample_names; }
    if (P.mode == 2) { region_alloc(&P, P.nwin); memset(P.first_occ, 0, P.nwin); region_print_header(&P, 3); }

    Region *sel = NULL; size_t n_sel = 0;
    if (bed_fn) {
        if (bed_read(bed_fn, &bf) == 0 && 1) {
            sel = bed_regions_merged(&B, &bf, &n_sel);
            if (P.mode == 0) { P.bed = bed_regions_merged(&B, &bf, &P.n_bed); P.bed_provided = 1; }
            else {
                P.raw_bed = bed_regions_raw(&B, &bf, &P.n_raw_bed); P.raw_bed_lines = bf.lines; P.n_raw_lines = bf.n_lines;
                if (bf.n_lines == 0) BAIL("empty BED file");
                region_alloc(&P, P.n_raw_bed); memset(P.first_occ, 1, P.n_raw_bed ? P.n_raw_bed : 1);
                /* isSortedAndNonOverlapping, depth.d:155-169 */
                P.general_collector = 0;
                for (size_t k = 0; k + 1 < P.n_raw_bed; k++) {
                    if (P.raw_bed[k].ref_id > P.raw_bed[k + 1].ref_id) { P.general_collector = 1; break; }
                    if (P.raw_bed[k].ref_id < P.raw_bed[k + 1].ref_id) continue;
                    if (P.raw_bed[k].end > P.raw_bed[k + 1].start) { P.general_collector = 1; break; }
                }
                /* header width = number of whitespace-separated fields of the first line */
                size_t nf = 0; { const char *l = bf.lines[0]; int in = 0; for (; *l; l++) { if (!is_white(*l)) { if (!in) { nf++; in = 1; } } else in = 0; } }
                region_print_header(&P, nf);
            }
        } else {
            char *ref = NULL; uint32_t beg, end; parse_region_string(bed_fn, &ref, &beg, &end);
            int id = bam_find_ref(&B, ref);
            if (id < 0) BAIL("couldn't open file %s or find reference %s", bed_fn, ref);
            if (end == UINT32_MAX) end = B.refs[id].length;
            sel = malloc(sizeof *sel); sel[0] = (Region){ (uint32_t)id, beg, end }; n_sel = 1;
            char *line = malloc(strlen(ref) + 40); sprintf(line, "%s\t%u\t%u", ref, beg, end);
            if (P.mode == 0) { P.bed = malloc(sizeof *P.bed); P.bed[0] = sel[0]; P.n_bed = 1; P.bed_provided = 1; }
            else {
                P.raw_bed = malloc(sizeof *P.raw_bed); P.raw_bed[0] = sel[0]; P.n_raw_bed = 1;
                P.raw_bed_lines = malloc(sizeof(char *)); P.raw_bed_lines[0] = line; P.n_raw_lines = 1;
                region_alloc(&P, 1); P.first_occ[0] = 1; P.general_collector = 0; region_print_header(&P, 3);
            }
            free(ref);
        }
    }

    ReadSrc src = { &B, B.first_rec, filter_mode, sel, n_sel, 0, -1, 0 };
    Sweep w; sweep_start(&w, &src);
    int last_ref_id = -2; t0 = now_s();
    while (!sweep_empty(&w)) {
        if (src.err) goto error;
        if (w.ref_id < 0 || w.ref_id >= B.n_ref) BAIL("read refers to reference #%d which is not in the header", w.ref_id);
        if (w.ref_id != last_ref_id) { last_ref_id = w.ref_id; fprintf(stderr, "Processing reference #%d (%s)\n", w.ref_id + 1, B.refs[w.ref_id].name); }
        if (P.mode == 0) base_push(&P, &w); else if (P.mode == 1) region_push(&P, &w); else window_push(&P, &w);
        g_stats.columns++;
        sweep_pop(&w);
    }
    if (src.err) goto error;
    if (P.mode == 0) base_close(&P);
    else if (P.mode == 1) { for (size_t id = 0; id < P.n_raw_bed; id++) for (int s = 0; s < P.n_sdata; s++) region_print_stats(&P, s, id); }
    else window_close(&P);
    g_stats.t_sweep = now_s() - t0;
    fflush(out); if (out_fn) fclose(out);
    free(w.reads); free(argv);
    return 0;
error:
    fprintf(stderr, "sambamba-depth: %s\n", g_err);
    if (out) fflush(out);
    (void)rc; free(argv);
    return 1;
}

/* --------------------------------------------- closed-form counter oracle
 * Per-read scatter restating the column semantics without iterating columns
 * (SURVEY 8a "closed form verified"): for every read passing the filter and
 * basesCovered()>0, walk the CIGAR from `pos`: M/=/X add to plane nt5(base) if
 * qual >= min_bq; D -> DEL; N -> REFSKIP.  Cross-checked against the sweep in
 * tests/test_oracle_golden.py.  A CIGAR that begins with N (quirk 1) is first turned
 * into what the sweep's cursor makes of it (closed_form_lead_n below).
 *
 * counts layout: [7][total_len] planes A,C,G,T,N,DEL,REFSKIP over the
 * concatenation of all references (ref_off[i] = sum of lengths before i).
 */
typedef struct { uint64_t n_records, n_pass, n_blocks, ulen, clen, covered, min_lin, max_lin; double t_inflate, t_scan; } ScatterStats;

/* Quirk 1 in closed form.  pread_init_cursor (pileup.d:175-192) steps over leading N operations without consuming them, so the
 * cursor walks the remaining operations that many columns early; past the last operation pread_increment (pileup.d:195-222) leaves
 * cur_op at the last operation it looked at -- cigar[n-1] -- for the columns that remain (the read stays in the sweep for
 * basesCovered() columns): base_process_current then counts a deletion if that operation is D and a reference skip if it does not
 * consume both query and reference.  Equivalent CIGAR: the leading N operations removed, their total length appended as N (or D).
 * If the last operation is M/=/X the sweep reads query offsets past l_seq there (pread_base's '=' / quality 0 stand in for the
 * reference's unchecked reads): not a defined result, left as it is -- the product refuses such a read.  Returns 1 if rewritten.
 * Checked against the faithful sweep in tests/test_oracle_golden.py. */
static int closed_form_lead_n(uint8_t *cig, uint32_t n_cigar) {
    uint32_t first = 0, k = 0; uint64_t nlead = 0; int found = 0;
    for (; first < n_cigar; first++) {
        uint32_t c = rd32(cig + 4 * first);
        if (!op_rcons(c)) continue;
        if ((c & 0xF) != 3) { found = 1; break; }
        nlead += op_len(c); k++;
    }
    if (!k || !found) return 0;
    uint32_t last = rd32(cig + 4 * (n_cigar - 1)) & 0xF;
    if (last == 0 || last == 7 || last == 8) return 0;
    uint32_t *tmp = malloc(4 * (size_t)n_cigar), w = 0;
    for (uint32_t j = 0; j < n_cigar; j++) { uint32_t c = rd32(cig + 4 * j); if (j < first && (c & 0xF) == 3) continue; tmp[w++] = c; }
    tmp[w++] = (uint32_t)(nlead << 4) | (last == 2 ? 2u : 3u);
    while (w < n_cigar) tmp[w++] = 6u;                       /* 0P: consumes nothing */
    for (uint32_t j = 0; j < n_cigar; j++) { uint32_t c = tmp[j]; cig[4 * j] = (uint8_t)c; cig[4 * j + 1] = (uint8_t)(c >> 8); cig[4 * j + 2] = (uint8_t)(c >> 16); cig[4 * j + 3] = (uint8_t)(c >> 24); }
    free(tmp);
    return 1;
}

/* One passing read of the closed form: scatter its CIGAR into the window (the body of the per-read loop; the record
 * walk that finds the reads is serial, the scatter runs on worker threads with relaxed atomic increments). */
typedef struct { const uint8_t *rec; uint64_t base, rlen; } ScatterRead;
typedef struct { const ScatterRead *rd; size_t n; _Atomic size_t *next; uint32_t *counts; uint64_t win_a, L; int min_bq; int atomic;
                 uint64_t n_seg; const uint64_t *seg_a, *seg_b; uint32_t *seg_reads; } ScatterJob;       /* optional: countRead per sorted, disjoint segment */
static void scatter_one(const ScatterJob *j, const ScatterRead *r) {
    const uint8_t *rec = r->rec; int32_t pos = (int32_t)rd32(rec + 4); uint32_t bmn = rd32(rec + 8), fnc = rd32(rec + 12);
    uint32_t l_name = bmn & 0xFF, n_cigar = fnc & 0xFFFF; int32_t l_seq = (int32_t)rd32(rec + 16);
    const uint8_t *cig = rec + 32 + l_name, *seq = cig + 4 * (size_t)n_cigar, *qual = seq + ((size_t)l_seq + 1) / 2;
    uint64_t base = r->base, rlen = r->rlen, p = (uint64_t)(uint32_t)pos, L = j->L, win_a = j->win_a; uint32_t q = 0; uint32_t *counts = j->counts;
    int64_t last_seg = -1;
    for (uint32_t i = 0; i < n_cigar; i++) {
        uint32_t c = rd32(cig + 4 * i), len = op_len(c), op = c & 0xF;
        if (op_match(c)) {
            if (j->n_seg) {       /* countRead (depth.d:661-669) in closed form: the read counts once in every segment in which it has a base with quality >= -q */
                uint64_t g0 = base + p, g1 = g0 + len; if (g1 > base + rlen) g1 = base + rlen;
                uint64_t lo = 0, hi = j->n_seg; while (lo < hi) { uint64_t m = (lo + hi) / 2; if (j->seg_b[m] <= g0) lo = m + 1; else hi = m; }
                for (uint64_t sgi = lo; sgi < j->n_seg && j->seg_a[sgi] < g1; sgi++) {
                    if ((int64_t)sgi <= last_seg) continue;
                    uint64_t xa = j->seg_a[sgi] > g0 ? j->seg_a[sgi] : g0, xb = j->seg_b[sgi] < g1 ? j->seg_b[sgi] : g1; int hit = 0;
                    for (uint64_t g = xa; g < xb && !hit; g++) { uint32_t qq = q + (uint32_t)(g - g0); if (qq < (uint32_t)l_seq && qual[qq] >= j->min_bq) hit = 1; }
                    if (hit) { __atomic_fetch_add(&j->seg_reads[sgi], 1u, __ATOMIC_RELAXED); last_seg = (int64_t)sgi; }
                }
            }
            for (uint32_t k = 0; k < len; k++, p++, q++) {
                if (p >= rlen || q >= (uint32_t)l_seq) continue;       /* clip at reference end (documented deviation for invalid input) */
                if (qual[q] < j->min_bq) continue;
                uint64_t g = base + p; if (g < win_a || g - win_a >= L) continue;
                uint8_t b = seq[q >> 1]; b = (q & 1) ? (b & 0xF) : (b >> 4);
                uint32_t *c32 = &counts[(uint64_t)NT16_TO_NT5[b] * L + (g - win_a)];
                if (j->atomic) __atomic_fetch_add(c32, 1u, __ATOMIC_RELAXED); else ++*c32;
            }
        } else if (op_rcons(c)) {
            int plane = (op == 2) ? 5 : 6;
            for (uint32_t k = 0; k < len; k++, p++) if (p < rlen) { uint64_t g = base + p; if (g >= win_a && g - win_a < L) { uint32_t *c32 = &counts[(uint64_t)plane * L + (g - win_a)]; if (j->atomic) __atomic_fetch_add(c32, 1u, __ATOMIC_RELAXED); else ++*c32; } }
        } else if (op_qcons(c)) q += len;
    }
}
static void *scatter_worker(void *arg) {
    ScatterJob *j = arg;
    for (;;) { size_t a = atomic_fetch_add(j->next, 4096), b = a + 4096 < j->n ? a + 4096 : j->n; if (a >= j->n) break; for (size_t i = a; i < b; i++) scatter_one(j, &j->rd[i]); }
    return NULL;
}

int oracle_bam_info(const char *bam_path, int *n_ref, uint64_t *total_len, uint64_t *ulen, uint64_t *n_blocks);
static int base_counts_impl(const char *bam_path, int mapq_gt, unsigned flag_reject, int min_bq, int nthreads, size_t max_file_bytes,
                            uint32_t *counts, uint64_t win_a, uint64_t win_len, ScatterStats *st, uint64_t n_seg, const uint64_t *seg_a, const uint64_t *seg_b, uint32_t *seg_reads) {
    Bam B; memset(&B, 0, sizeof B);
    double t0 = now_s();
    if (bgzf_load(&B.z, bam_path, nthreads, max_file_bytes)) return -1;
    double t1 = now_s();
    if (bam_parse_header(&B, max_file_bytes != 0)) return -1;
    uint64_t total = 0; uint64_t *ref_off = calloc(B.n_ref + 1, sizeof *ref_off);
    for (int i = 0; i < B.n_ref; i++) { ref_off[i] = total; total += B.refs[i].length; } ref_off[B.n_ref] = total;
    uint64_t nrec = 0, npass = 0; size_t off = B.first_rec; const uint8_t *u = B.z.u;
    uint64_t L = win_len, min_lin = UINT64_MAX, max_lin = 0;
    ScatterRead *rd = NULL; size_t nrd = 0, cap = 0;
    while (off + 4 <= B.z.ulen) {
        uint32_t bs = rd32(u + off); if (off + 4 + (size_t)bs > B.z.ulen) break;
        const uint8_t *rec = u + off + 4; off += 4 + (size_t)bs; nrec++;
        int32_t ref_id = (int32_t)rd32(rec), pos = (int32_t)rd32(rec + 4); uint32_t bmn = rd32(rec + 8), fnc = rd32(rec + 12);
        uint32_t l_name = bmn & 0xFF, mapq = (bmn >> 8) & 0xFF, flag = fnc >> 16, n_cigar = fnc & 0xFFFF;
        if (!((int)mapq > mapq_gt) || (flag & flag_reject) || (flag & 0x4) || ref_id < 0 || ref_id >= B.n_ref) continue;
        const uint8_t *cig = rec + 32 + l_name;
        uint64_t span = 0; for (uint32_t i = 0; i < n_cigar; i++) { uint32_t c = rd32(cig + 4 * i); if (op_rcons(c)) span += op_len(c); }
        if (!span) continue;
        npass++;
        /* (B.z.u is this call's own copy of the inflated stream.)  Region / window statistics take readCount and meanCoverage from the CIGAR
         * as written (countOverlappingBases, depth.d:671-698) and the percentages from the cursor: no closed form here, only the sweep knows */
        if (closed_form_lead_n((uint8_t *)cig, n_cigar) && n_seg) { free(rd); free(ref_off); bgzf_free(&B.z); return fail("closed form of the region statistics: a CIGAR that begins with N is not modelled (use the sweep)"); }
        { uint64_t g0 = ref_off[ref_id] + (uint32_t)pos, g1 = g0 + span; if (g0 < min_lin) min_lin = g0; if (g1 > max_lin) max_lin = g1; }
        if (!counts) continue;
        if (nrd == cap) { cap = cap ? cap * 2 : (1u << 16); rd = realloc(rd, cap * sizeof *rd); }
        rd[nrd].rec = rec; rd[nrd].base = ref_off[ref_id]; rd[nrd].rlen = B.refs[ref_id].length; nrd++;
    }
    if (counts && nrd) {
        _Atomic size_t next = 0; int nt = nthreads > 1 ? nthreads : 1;
        ScatterJob job = { rd, nrd, &next, counts, win_a, L, min_bq, nt > 1, n_seg, seg_a, seg_b, seg_reads };
        if (nt == 1) scatter_worker(&job);
        else { pthread_t *th = calloc(nt, sizeof *th); for (int t = 0; t < nt; t++) pthread_create(&th[t], NULL, scatter_worker, &job); for (int t = 0; t < nt; t++) pthread_join(th[t], NULL); free(th); }
    }
    free(rd);
    if (st) {
        st->n_records = nrec; st->n_pass = npass; st->n_blocks = B.z.n_blocks; st->ulen = B.z.ulen; st->clen = B.z.file_len; st->t_inflate = t1 - t0; st->t_scan = now_s() - t1; st->covered = 0;
        st->min_lin = min_lin; st->max_lin = max_lin;
        if (counts) { uint64_t cv = 0; for (uint64_t i = 0; i < L; i++) { uint32_t s = 0; for (int k = 0; k < 7; k++) s += counts[(uint64_t)k * L + i]; cv += s > 0; } st->covered = cv; }
    }
    free(ref_off); bgzf_free(&B.z);
    return 0;
}

int oracle_base_counts(const char *bam_path, int mapq_gt, unsigned flag_reject, int min_bq, int nthreads, size_t max_file_bytes,
                       uint32_t *counts /* [7][win_len], may be NULL to just scan */, uint64_t win_a /* first linear position of the window */, uint64_t win_len, ScatterStats *st) {
    return base_counts_impl(bam_path, mapq_gt, flag_reject, min_bq, nthreads, max_file_bytes, counts, win_a, win_len, st, 0, NULL, NULL, NULL);
}

/* Region / window statistics in closed form (PerSampleRegionData, depth.d:609-635, as printRegionStats :847-876 uses them), for
 * segments [seg_a[i], seg_b[i]) in linear coordinates, sorted and disjoint (BED regions, or the tiling windows of `depth window`
 * without --overlap): n_reads = reads with at least one M/=/X base of quality >= -q inside (countRead :661-669), n_bases = sum of
 * the A,C,G,T,N counters, cov[t][i] = positions whose COV (all seven counters) reaches thr[t].  Checked against the faithful
 * sweep's region and window output in tests/test_oracle_golden.py; used by bench.py to verify full-size window / region runs,
 * where the serial sweep would take minutes.  One sample, no -m.  Test infrastructure only. */
typedef struct { const uint32_t *counts; uint64_t L; uint64_t n_seg; const uint64_t *a, *b; uint32_t n_thr; const uint32_t *thr; uint32_t *bases, *cov; _Atomic uint64_t *next; } SegSumJob;
static void *seg_sum_worker(void *arg) {
    SegSumJob *j = arg;
    for (;;) {
        uint64_t i0 = atomic_fetch_add(j->next, 256), i1 = i0 + 256 < j->n_seg ? i0 + 256 : j->n_seg; if (i0 >= j->n_seg) break;
        for (uint64_t i = i0; i < i1; i++) {
            uint64_t nb = 0;
            for (uint64_t g = j->a[i]; g < j->b[i] && g < j->L; g++) {
                uint32_t s5 = 0, s7 = 0; for (int k = 0; k < 7; k++) { uint32_t v = j->counts[(uint64_t)k * j->L + g]; s7 += v; if (k < 5) s5 += v; }
                nb += s5;
                for (uint32_t t = 0; t < j->n_thr; t++) if (s7 >= j->thr[t] && s7) j->cov[(uint64_t)t * j->n_seg + i]++;
            }
            j->bases[i] = (uint32_t)nb;
        }
    }
    return NULL;
}
int oracle_segment_stats(const char *bam_path, int mapq_gt, unsigned flag_reject, int min_bq, int nthreads, uint64_t n_seg, const uint64_t *seg_a, const uint64_t *seg_b,
                         uint32_t n_thr, const uint32_t *thr, uint32_t *out_reads, uint32_t *out_bases, uint32_t *out_cov /* [n_thr][n_seg] */) {
    int n_ref; uint64_t total, ulen, nblk;
    if (oracle_bam_info(bam_path, &n_ref, &total, &ulen, &nblk)) return -1;
    uint32_t *counts = calloc((size_t)7 * (total ? total : 1), 4); if (!counts) { snprintf(g_err, sizeof g_err, "out of memory for %llu positions", (unsigned long long)total); return -1; }
    memset(out_reads, 0, n_seg * 4); memset(out_bases, 0, n_seg * 4); if (n_thr) memset(out_cov, 0, (size_t)n_thr * n_seg * 4);
    int rc = base_counts_impl(bam_path, mapq_gt, flag_reject, min_bq, nthreads, 0, counts, 0, total, NULL, n_seg, seg_a, seg_b, out_reads);
    if (!rc && n_seg) {
        _Atomic uint64_t next = 0; int nt = nthreads > 1 ? nthreads : 1;
        SegSumJob job = { counts, total, n_seg, seg_a, seg_b, n_thr, thr, out_bases, out_cov, &next };
        if (nt == 1) seg_sum_worker(&job);
        else { pthread_t *th = calloc(nt, sizeof *th); for (int t = 0; t < nt; t++) pthread_create(&th[t], NULL, seg_sum_worker, &job); for (int t = 0; t < nt; t++) pthread_join(th[t], NULL); free(th); }
    }
    free(counts);
    return rc;
}

/* --------------------------------------------- closed form for -m (fix-mate-overlaps), base mode
 * The sweep (base_write_column above, depth.d:495-556 with detectOverlappingMates :319-388 and selectBetterMate
 * :391-399) counts, in every column, each PAIR of same-name reads once: only the better mate contributes (either on
 * a D/N there -> the one with the higher MAPQ, second on ties; else the one with the higher base quality, second on
 * ties).  Pairs are adjacent entries of the column's reads sorted by (name hash, arrival order), so of three
 * same-name reads present in a column the first two pair up and the third counts alone.  Reads that are not in a
 * pair in a column count as usual (state none/past).  Restated per name group instead of per column of the whole
 * file: start from the plain closed form, then, for every group of same-name reads, walk the columns where at
 * least two of them are present and take the loser's contribution out again.
 * Cross-checked against the sweep in tests/test_oracle_golden.py.  Test infrastructure only. */
typedef struct { uint64_t h; uint32_t idx; } MateKey;
static int mate_key_cmp(const void *a, const void *b) { const MateKey *x = a, *y = b; if (x->h != y->h) return x->h < y->h ? -1 : 1; return x->idx < y->idx ? -1 : (x->idx > y->idx); }

int oracle_base_counts_fix_mates(const char *bam_path, int mapq_gt, unsigned flag_reject, int min_bq,
                                 uint32_t *counts /* [7][win_len] */, uint64_t win_a, uint64_t win_len, uint64_t *n_pair_columns) {
    if (oracle_base_counts(bam_path, mapq_gt, flag_reject, min_bq, 1, 0, counts, win_a, win_len, NULL)) return -1;
    Bam B; memset(&B, 0, sizeof B);
    if (bgzf_load(&B.z, bam_path, 1, 0)) return -1;
    if (bam_parse_header(&B, 0)) return -1;
    uint64_t *ref_off = calloc(B.n_ref + 1, sizeof *ref_off); { uint64_t t = 0; for (int i = 0; i < B.n_ref; i++) { ref_off[i] = t; t += B.refs[i].length; } }
    PRead *rd = NULL; size_t n = 0, cap = 0;
    size_t off = B.first_rec; const uint8_t *u = B.z.u;
    while (off + 4 <= B.z.ulen) {
        uint32_t bs = rd32(u + off); if (off + 4 + (size_t)bs > B.z.ulen) break;
        PRead r; if (parse_record(&B, u + off + 4, bs, &r)) { free(rd); free(ref_off); return -1; }
        off += 4 + (size_t)bs;
        if (!((int)r.mapq > mapq_gt) || (r.flag & flag_reject) || (r.flag & 0x4) || r.ref_id < 0 || r.ref_id >= B.n_ref || bases_covered(&r) <= 0) continue;
        if (n == cap) { cap = cap ? cap * 2 : 1024; rd = realloc(rd, cap * sizeof *rd); }
        rd[n++] = r;
    }
    MateKey *key = malloc((n ? n : 1) * sizeof *key);
    for (size_t i = 0; i < n; i++) { key[i].h = rd[i].name_hash; key[i].idx = (uint32_t)i; }
    qsort(key, n, sizeof *key, mate_key_cmp);
    uint64_t pair_cols = 0; const uint64_t L = win_len;
    for (size_t g0 = 0; g0 < n;) {
        size_t g1 = g0 + 1; while (g1 < n && key[g1].h == key[g0].h) g1++;
        size_t gn = g1 - g0;
        if (gn >= 2) {
            /* members in arrival (file) order; cursors start when the column reaches a member's start */
            PRead **m = malloc(gn * sizeof *m); uint8_t *started = calloc(gn, 1);
            int64_t lo = INT64_MAX, hi = 0;
            for (size_t k = 0; k < gn; k++) { m[k] = &rd[key[g0 + k].idx]; int64_t a = (int64_t)(ref_off[m[k]->ref_id] + (uint32_t)m[k]->pos), b = (int64_t)(ref_off[m[k]->ref_id] + m[k]->end_pos); if (a < lo) lo = a; if (b > hi) hi = b; }
            for (int64_t g = lo; g < hi; g++) {
                PRead *pres[64]; size_t np = 0;
                for (size_t k = 0; k < gn; k++) {
                    int64_t a = (int64_t)(ref_off[m[k]->ref_id] + (uint32_t)m[k]->pos), b = (int64_t)(ref_off[m[k]->ref_id] + m[k]->end_pos);
                    if (g < a || g >= b) continue;
                    if (!started[k]) { pread_init_cursor(m[k]); started[k] = 1; } else pread_increment(m[k]);
                    if (np < 64) pres[np++] = m[k];
                }
                /* detectOverlappingMates restricted to this name: adjacent pairs in arrival order; the read left over
                 * (or alone) goes to `past` if it had been flagged -- unless it is the very last entry of the column's
                 * hash-sorted array AND its predecessor has the same hash (depth.d:380-384), in which case it keeps its
                 * state.  A read in state `detected` is skipped by the plain loop, every pair adds its better mate. */
                PRead *pa[32], *pb[32]; size_t npairs = 0;
                for (size_t i = 0; i < np;) {
                    if (i + 1 < np) {
                        PRead *r1 = pres[i], *r2 = pres[i + 1];
                        if (r1->sample_id == r2->sample_id && r1->l_read_name == r2->l_read_name && !memcmp(r1->name, r2->name, r1->l_read_name)) {
                            if (npairs < 32) { pa[npairs] = r1; pb[npairs] = r2; npairs++; }
                            if (r1->mate_overlap == MO_NONE) r1->mate_overlap = MO_DETECTED;
                            if (r2->mate_overlap == MO_NONE) r2->mate_overlap = MO_DETECTED;
                            i += 2; continue;
                        }
                        i += 1; continue;          /* same hash, different name: the reference moves on without touching the state */
                    }
                    /* the last present read of this name, not consumed by a pair */
                    PRead *r = pres[i];
                    if (r->mate_overlap != MO_NONE) {
                        int keep = 0;
                        if (np >= 2) {               /* its predecessor in the sorted array has the same hash: `past` only if something follows it */
                            int follows = 0;
                            for (size_t q = 0; q < n && !follows; q++) {
                                const PRead *o = &rd[q];
                                if (o->name_hash <= r->name_hash || o->ref_id != r->ref_id) continue;
                                int64_t a = (int64_t)(ref_off[o->ref_id] + (uint32_t)o->pos), b = (int64_t)(ref_off[o->ref_id] + o->end_pos);
                                if (g >= a && g < b) follows = 1;
                            }
                            keep = !follows;
                        }
                        if (!keep) r->mate_overlap = MO_PAST;
                    }
                    i += 1;
                }
                if (npairs) pair_cols += npairs;
                if (g >= (int64_t)win_a && (uint64_t)(g - (int64_t)win_a) < L) {
                    uint64_t x = (uint64_t)(g - (int64_t)win_a);
                    /* the plain closed form counted every present read once; take out what the sweep does not count
                     * (reads in state `detected`) and add what it counts on top (the better mate of every pair) */
                    for (size_t k = 0; k < np; k++) if (pres[k]->mate_overlap == MO_DETECTED) {
                        char c = pread_base(pres[k]);
                        if (c == '-') counts[(uint64_t)(((pres[k]->cur_op & 0xF) == 2) ? 5 : 6) * L + x]--;
                        else if (pread_qual(pres[k]) >= min_bq) counts[(uint64_t)base5_of_char(c) * L + x]--;
                    }
                    for (size_t k = 0; k < npairs; k++) {
                        PRead *w = select_better_mate(pa[k], pb[k]); char c = pread_base(w);
                        if (c == '-') counts[(uint64_t)(((w->cur_op & 0xF) == 2) ? 5 : 6) * L + x]++;
                        else if (pread_qual(w) >= min_bq) counts[(uint64_t)base5_of_char(c) * L + x]++;
                    }
                }
            }
            free(m); free(started);
        }
        g0 = g1;
    }
    if (n_pair_columns) *n_pair_columns = pair_cols;
    free(key); free(rd); free(ref_off); bgzf_free(&B.z);
    return 0;
}

/* header info for Python tests */
int oracle_bam_info(const char *bam_path, int *n_ref, uint64_t *total_len, uint64_t *ulen, uint64_t *n_blocks) {
    Bam B; memset(&B, 0, sizeof B);
    if (bgzf_load(&B.z, bam_path, 1, 0)) return -1;
    if (bam_parse_header(&B, 0)) return -1;
    uint64_t t = 0; for (int i = 0; i < B.n_ref; i++) t += B.refs[i].length;
    *n_ref = B.n_ref; *total_len = t; *ulen = B.z.ulen; *n_blocks = B.z.n_blocks;
    bgzf_free(&B.z); return 0;
}
/* inflate whole file into caller buffer (for K1 parity) */
int64_t oracle_inflate_file(const char *bam_path, uint8_t *dst, uint64_t cap) {
    Bgzf z; if (bgzf_load(&z, bam_path, 1, 0)) return -1;
    int64_t n = (int64_t)z.ulen; if (dst) { if (cap < z.ulen) { bgzf_free(&z); return -2; } memcpy(dst, z.u, z.ulen); }
    bgzf_free(&z); return n;
}
void oracle_get_stats(double *t_inflate, double *t_sweep, uint64_t *columns, uint64_t *file_bytes) { *t_inflate = g_stats.t_inflate; *t_sweep = g_stats.t_sweep; *columns = g_stats.columns; *file_bytes = g_stats.file_bytes; }


/* ------------------------------------------------------------------ BAI builder (sambamba index; SURVEY 8f rank 2)
 * A restatement of IndexBuilder (BioD/bio/std/hts/bam/bai/indexing.d:56-351, createIndex :356-366) over the virtual offsets the
 * reference's stream reports (BgzfInputStream: a position at the end of a member is the start of the next one, inputstream.d:430-452,
 * :508-530; after the last member it is the offset of the EOF marker).  put() :290-333: reads are taken in file order; a read without
 * reference or with position < 0 only counts in the metadata; the previous read's linear-index entries (:133-161) and, when the bin
 * changes or a new reference begins, its chunk (:219-246: merged with the bin's last chunk when that one ends in the same member) are
 * flushed when the next read arrives.  dumpCurrentReference :184-216 writes the bins, the metadata pseudo-bin 37450 and the linear
 * index with its gaps filled from the left (:163-182).
 * One deviation, stated: the reference writes a reference's bins in the iteration order of a D associative array (:188), which is not
 * defined by anything but that runtime; this restatement writes them in ascending bin number.  A reader of the index cannot tell.
 * Returns the size of the index (written to out when cap suffices), or -1 (oracle_last_error()).                                       */
typedef struct { uint64_t beg, end; } BaiChunkO;
typedef struct { uint32_t bin; BaiChunkO *c; size_t n, cap; } BaiBinO;
typedef struct { uint8_t *p; size_t n, cap; } OutBuf;
static void ob_put(OutBuf *o, const void *src, size_t len) { if (o->n + len > o->cap) { o->cap = (o->n + len) * 2 + 4096; o->p = realloc(o->p, o->cap); } memcpy(o->p + o->n, src, len); o->n += len; }
static void ob_u32(OutBuf *o, uint32_t v) { uint8_t b[4] = { (uint8_t)v, (uint8_t)(v >> 8), (uint8_t)(v >> 16), (uint8_t)(v >> 24) }; ob_put(o, b, 4); }
static void ob_u64(OutBuf *o, uint64_t v) { ob_u32(o, (uint32_t)v); ob_u32(o, (uint32_t)(v >> 32)); }
static int bin_cmp(const void *a, const void *b) { const BaiBinO *x = a, *y = b; return x->bin < y->bin ? -1 : x->bin > y->bin; }
static uint64_t voffset_of(const Bgzf *z, uint64_t u) {      /* virtualTell() at inflated offset u */
    if (u >= z->ulen) { const BgzfBlock *l = &z->blocks[z->n_blocks - 1]; return (l->coff + l->bsize) << 16; }
    size_t lo = 0, hi = z->n_blocks; while (lo + 1 < hi) { size_t m = (lo + hi) / 2; if (z->blocks[m].uoff <= u) lo = m; else hi = m; }
    return (z->blocks[lo].coff << 16) | (u - z->blocks[lo].uoff);
}
#define BAI_LIN_N 32769           /* BAI_MAX_BIN_ID - BAI_MAX_NONLEAF_BIN_ID + 1, indexing.d:279 */
static size_t lin_off(int32_t pos) { return pos < 0 ? 0 : (size_t)pos / 16384; }      /* toLinearIndexOffset :51-53 */
typedef struct {
    OutBuf out; uint64_t *lin; size_t lin_len;
    int first_read; int32_t p_ref, p_pos, p_end; uint32_t p_bin; int p_unmapped; uint64_t p_svo, p_evo;      /* _prev_read */
    uint64_t no_coord, beg_vo, end_vo, unmapped, mapped, cur_beg;
    BaiBinO *bins; size_t n_bins, cap_bins;
} BaiB;
static void bb_update_linear(BaiB *b) {                      /* :133-161 */
    size_t beg = lin_off(b->p_pos), end = b->p_unmapped ? beg : lin_off(b->p_pos + (b->p_end - b->p_pos) - 1);
    for (size_t i = beg; i <= end && i < BAI_LIN_N; i++) if (b->lin[i] == 0) b->lin[i] = b->p_svo;
    if (end + 1 > b->lin_len) b->lin_len = end + 1;
}
static void bb_update_chunks(BaiB *b) {                      /* :219-246 */
    BaiBinO *bn = NULL;
    for (size_t i = 0; i < b->n_bins; i++) if (b->bins[i].bin == b->p_bin) bn = &b->bins[i];
    if (!bn) { BaiBinO nb = { b->p_bin, NULL, 0, 0 }; VEC_PUSH(b->bins, b->n_bins, b->cap_bins, nb); bn = &b->bins[b->n_bins - 1]; }
    if (bn->n == 0 || (bn->c[bn->n - 1].end >> 16) != (b->cur_beg >> 16)) { BaiChunkO c = { b->cur_beg, b->p_evo }; VEC_PUSH(bn->c, bn->n, bn->cap, c); }
    else bn->c[bn->n - 1].end = b->p_evo;
    b->cur_beg = b->p_evo;
}
static void bb_dump_reference(BaiB *b) {                     /* :184-216 */
    qsort(b->bins, b->n_bins, sizeof *b->bins, bin_cmp);
    ob_u32(&b->out, (uint32_t)(b->n_bins + 1));
    for (size_t i = 0; i < b->n_bins; i++) {
        ob_u32(&b->out, b->bins[i].bin); ob_u32(&b->out, (uint32_t)b->bins[i].n);
        for (size_t k = 0; k < b->bins[i].n; k++) { ob_u64(&b->out, b->bins[i].c[k].beg); ob_u64(&b->out, b->bins[i].c[k].end); }
        free(b->bins[i].c);
    }
    ob_u32(&b->out, 37450); ob_u32(&b->out, 2); ob_u64(&b->out, b->beg_vo); ob_u64(&b->out, b->end_vo); ob_u64(&b->out, b->mapped); ob_u64(&b->out, b->unmapped);
    ob_u32(&b->out, (uint32_t)b->lin_len);
    uint64_t last = 0;
    for (size_t i = 0; i < b->lin_len; i++) { uint64_t v = i < BAI_LIN_N ? b->lin[i] : 0; if (v == 0) v = last; else last = v; ob_u64(&b->out, v); }
    memset(b->lin, 0, BAI_LIN_N * sizeof *b->lin); b->lin_len = 0; b->n_bins = 0;
    b->cur_beg = b->p_evo; b->beg_vo = b->end_vo = b->cur_beg; b->unmapped = b->mapped = 0;
}
int64_t oracle_build_bai(const char *bam_path, uint8_t *out, uint64_t cap, int nthreads) {
    Bam B; memset(&B, 0, sizeof B);
    if (bgzf_load(&B.z, bam_path, nthreads, 0)) return -1;
    if (bam_parse_header(&B, 0)) return -1;
    BaiB b; memset(&b, 0, sizeof b); b.lin = calloc(BAI_LIN_N, sizeof *b.lin); b.first_read = 1; b.p_ref = -1; b.beg_vo = UINT64_MAX;
    ob_put(&b.out, "BAI\1", 4); ob_u32(&b.out, (uint32_t)B.n_ref);
    size_t off = B.first_rec; const uint8_t *u = B.z.u; int rc = 0;
    while (off + 4 <= B.z.ulen) {
        uint32_t bs = rd32(u + off); if (off + 4 + (size_t)bs > B.z.ulen) { rc = fail("not enough data in stream"); break; }
        PRead r; if (parse_record(&B, u + off + 4, bs, &r)) { rc = -1; break; }
        const uint64_t svo = voffset_of(&B.z, off), evo = voffset_of(&B.z, off + 4 + bs);
        off += 4 + (size_t)bs;
        const uint32_t bin = rd32(r.rec + 8) >> 16; const int unm = (r.flag & 0x4) != 0; const int32_t endp = r.pos + bases_covered(&r);
        /* checkThatInputIsSorted :259-271 */
        if (!b.first_read && r.ref_id != -1 && !(b.p_ref < r.ref_id) && !(r.ref_id == b.p_ref && r.pos >= b.p_pos)) { rc = fail("BAM file is not coordinate-sorted: read '%s' (%d:%d) must be after the previous read (%d:%d)", r.name, r.ref_id, r.pos, b.p_ref, b.p_pos); break; }
        if (r.ref_id >= 0 && r.pos >= 0) {
            if (b.first_read) {                              /* :301-311 */
                b.first_read = 0; b.cur_beg = svo;
                for (int i = 0; i < r.ref_id; i++) { ob_u32(&b.out, 0); ob_u32(&b.out, 0); }
            } else {
                if (r.ref_id > b.p_ref) {                    /* :316-323 */
                    bb_update_linear(&b); bb_update_chunks(&b); bb_dump_reference(&b);
                    for (int i = b.p_ref + 1; i < r.ref_id; i++) { ob_u32(&b.out, 0); ob_u32(&b.out, 0); }
                } else if (r.ref_id == b.p_ref) {            /* :325-330 */
                    bb_update_linear(&b);
                    if (bin != b.p_bin) bb_update_chunks(&b);
                }
            }
            b.p_ref = r.ref_id; b.p_pos = r.pos; b.p_end = endp; b.p_bin = bin; b.p_unmapped = unm; b.p_svo = svo; b.p_evo = evo;      /* updateLastReadInfo */
        }
        /* scope(exit) updateMetadata :117-131 */
        if (r.ref_id == -1) b.no_coord++;
        else { if (unm) b.unmapped++; else b.mapped++; if (b.beg_vo == UINT64_MAX) b.beg_vo = svo; b.end_vo = evo; }
    }
    if (!rc) {                                               /* finish :336-350 */
        if (!b.first_read) { bb_update_linear(&b); bb_update_chunks(&b); bb_dump_reference(&b); }
        for (int i = b.p_ref + 1; i < B.n_ref; i++) { ob_u32(&b.out, 0); ob_u32(&b.out, 0); }
        ob_u64(&b.out, b.no_coord);
    }
    int64_t n = rc ? -1 : (int64_t)b.out.n;
    if (!rc && out && cap >= b.out.n) memcpy(out, b.out.p, b.out.n);
    free(b.out.p); free(b.lin); free(b.bins); bgzf_free(&B.z);
    return n;
}

#ifdef ORACLE_MAIN
int main(int argc, char **argv) {
    /* usage: depth_oracle [--inflate-threads N] [--max-file-bytes B] depth base|region|window ... ; prints timing to stderr with --stats */
    int ith = 0, stats = 0; size_t maxb = 0; int i = 1;
    while (i < argc) {
        if (!strcmp(argv[i], "--inflate-threads") && i + 1 < argc) { ith = atoi(argv[i + 1]); i += 2; }
        else if (!strcmp(argv[i], "--max-file-bytes") && i + 1 < argc) { maxb = strtoull(argv[i + 1], NULL, 10); i += 2; }
        else if (!strcmp(argv[i], "--stats")) { stats = 1; i++; }
        else break;
    }
    if (i < argc && !strcmp(argv[i], "depth")) i++;
    static char obuf[1 << 20]; setvbuf(stdout, obuf, _IOFBF, sizeof obuf);
    /* depth_main expects args[0]=prog, args[1]=mode */
    int rc = oracle_depth_main(argc - i + 1, argv + i - 1, stdout, ith, maxb);
    fflush(stdout);
    if (stats) fprintf(stderr, "{\"t_inflate\": %.6f, \"t_sweep\": %.6f, \"columns\": %llu, \"file_bytes\": %llu}\n", g_stats.t_inflate, g_stats.t_sweep, (unsigned long long)g_stats.columns, (unsigned long long)g_stats.file_bytes);
    return rc;
}
#endif
