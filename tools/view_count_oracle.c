/* view_count_oracle.c -- CPU restatement of `sambamba view -c` and of `sambamba view`'s SAM lines and JSON records (TEST INFRASTRUCTURE: the checker the GPU
 * count and text are compared with).
 *
 * What is restated (sambamba/view.d:265-379), record by record, without shortcuts:
 *   - FlagBitFilter (utils/common/filtering.d:176-187) and SubsampleFilter (:340-371, FNV-1a 64 over the name, then the seed's 8 bytes);
 *   - -L on a file that is not SO:coordinate: BedFilter (:118-160), its interval-tree overlap rule iv.stop > start && iv.start < stop on
 *     unsigned coordinates (utils/common/intervaltree.d:122-131), checked against every region of the read's reference;
 *   - -L on a sorted file: getReadsOverlapping (randomaccessmanager.d:316-338) -- regions grouped by reference, each group walked by the
 *     BamReadFilter state machine (:366-462) over the file's records;
 *   - positional regions: one BamReadFilter with one region per argument, the streams joined; '*' is unmappedReads (reader.d:370-391): skip to
 *     the first record with refID -1, then every record to the end of the file.
 * The record streams are the file's records in order, not the BAI chunks the reference reads: on a coordinate-sorted file with a correct index
 * the state machine selects the same reads from either, and this file does not depend on the engine's index code.  -F is not restated here:
 * the tests apply a Python statement of the query and count the reduced file.
 *
 * The SAM line of a selected read is a literal C statement of BamRead.toSam (BioD/bio/std/hts/bam/read.d:695-760) plus '\n'
 * (alignmentrangeprocessor.d:72-75), with the tag values of tagvalue.d:468-504 and floats through snprintf("%g", (double)f) as
 * bio/core/utils/format.d:92-134 does.  Where the reference throws or indexes out of bounds (an unknown tag type, a tag running past the record,
 * a Z / H value without its NUL, a reference ID outside [-1, n_ref) that is printed), the text entry point returns an error.
 * The JSON record of `view -f json` is a literal C statement of BamRead.toJson (read.d:768-830) plus '\n' with BioD's writers: writeStringJson and
 * its escape table, writeFloatJson (%g, +-1.0e+1024 for +-inf, null for NaN) and itoa (format.d:66-87,196-270); its refusals are the SAM line's.
 * -v is a literal C statement of BioD's isValid (bio/std/hts/bam/validation/alignment.d:138-562), applied in view_main's filter chain: after
 * SubsampleFilter, before FlagBitFilter and -F, and before BedFilter; where its tag walk throws or reads past the record, the run fails.
 * Library: view_count_oracle(), view_text_oracle(), view_json_oracle(), view_text_oracle_free(), view_count_oracle_hash(),
 * view_count_oracle_error(), view_count_oracle_set_valid() (-v for the calls that follow), view_valid_oracle() (one record).  With -DORACLE_MAIN
 * also a CLI:
 *   view_count_oracle view [-c] [-v] [-f sam|json] [--num-filter=I1/I2] [-s FRAC] [--subsampling-seed=SEED] [-L BED] in.bam [region ...]
 * which prints the count as `sambamba view -c` does, or without -c the SAM lines or JSON records (no header), or "sambamba-view: <msg>" and exit
 * code 1 for the errors it restates. */
#include <ctype.h>
#include <errno.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

static char g_err[512];
const char* view_count_oracle_error(void) { return g_err; }

typedef struct { int32_t ref, pos; uint16_t flag; int64_t bc; const uint8_t* name; uint32_t l_name; const uint8_t* p; uint32_t bs; } Rec;      /* p: the refID field, bs: block_size */
typedef struct { uint8_t* u; size_t n; int n_ref; char** names; int sorted; Rec* r; size_t nr; } Bam;

static uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

static void bam_free(Bam* b) {
    if (b->names) for (int i = 0; i < b->n_ref; i++) free(b->names[i]);
    free(b->names); free(b->u); free(b->r); memset(b, 0, sizeof *b);
}

static int bam_load(const char* path, Bam* b) {
    memset(b, 0, sizeof *b);
    gzFile f = gzopen(path, "rb");
    if (!f) { snprintf(g_err, sizeof g_err, "Cannot open file `%s' in mode `rb' (%s)", path, strerror(errno)); return -1; }
    size_t cap = 1 << 20; b->u = malloc(cap);
    for (;;) {
        if (b->n == cap) { cap *= 2; b->u = realloc(b->u, cap); }
        int k = gzread(f, b->u + b->n, (unsigned)(cap - b->n > (1u << 30) ? (1u << 30) : cap - b->n));
        if (k < 0) { int e; snprintf(g_err, sizeof g_err, "DEFLATE error: %s", gzerror(f, &e)); gzclose(f); return -1; }
        if (k == 0) break;
        b->n += (size_t)k;
    }
    gzclose(f);
    const uint8_t* u = b->u; size_t n = b->n;
    if (n < 12 || memcmp(u, "BAM\1", 4)) { snprintf(g_err, sizeof g_err, "Invalid file format: expected BAM\\1"); return -1; }
    uint32_t l_text = rd32(u + 4); size_t o = 8 + (size_t)l_text;
    if (o + 4 > n) { snprintf(g_err, sizeof g_err, "truncated BAM header"); return -1; }
    {   /* @HD SO:coordinate */
        const char* t = (const char*)u + 8; size_t i = 0;
        while (i < l_text) {
            size_t e = i; while (e < l_text && t[e] != '\n') e++;
            if (e - i >= 3 && !memcmp(t + i, "@HD", 3)) for (size_t k = i; k + 14 <= e; k++) if (!memcmp(t + k, "\tSO:coordinate", 14) && (k + 14 == e || t[k + 14] == '\t')) b->sorted = 1;
            i = e + 1;
        }
    }
    b->n_ref = (int)rd32(u + o); o += 4;
    b->names = calloc((size_t)b->n_ref + 1, sizeof(char*));
    for (int i = 0; i < b->n_ref; i++) {
        uint32_t ln = rd32(u + o); b->names[i] = malloc(ln + 1); memcpy(b->names[i], u + o + 4, ln); b->names[i][ln] = 0; o += 8 + ln;
    }
    size_t rcap = 1024; b->r = malloc(rcap * sizeof(Rec));
    while (o + 4 <= n) {
        uint32_t bs = rd32(u + o);
        if (o + 4 + bs > n) { snprintf(g_err, sizeof g_err, "not enough data in stream"); return -1; }
        const uint8_t* p = u + o + 4;
        if (b->nr == rcap) { rcap *= 2; b->r = realloc(b->r, rcap * sizeof(Rec)); }
        Rec* x = &b->r[b->nr++];
        x->ref = (int32_t)rd32(p); x->pos = (int32_t)rd32(p + 4);
        uint32_t bmn = rd32(p + 8), fnc = rd32(p + 12);
        x->l_name = bmn & 0xFF; x->flag = (uint16_t)(fnc >> 16); x->p = p; x->bs = bs;
        uint32_t nc = fnc & 0xFFFF; x->name = p + 32;
        x->bc = 0;
        if (!(x->flag & 4)) for (uint32_t k = 0; k < nc; k++) { uint32_t c = rd32(p + 32 + x->l_name + 4 * k), op = c & 15; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) x->bc += c >> 4; }      /* basesCovered, read.d:255-262 */
        o += 4 + bs;
    }
    if (n - o >= 4) { snprintf(g_err, sizeof g_err, "not enough data in stream"); return -1; }
    return 0;
}

uint64_t view_count_oracle_hash(const uint8_t* name, size_t len, uint64_t seed) {
    uint64_t h = 14695981039346656037ull;
    for (size_t i = 0; i < len; i++) { h ^= name[i]; h *= 1099511628211ull; }
    for (int i = 0; i < 8; i++) { h ^= (seed >> (8 * i)) & 0xFF; h *= 1099511628211ull; }
    return h;
}

typedef struct { uint32_t ref, start, end; } Reg;

/* Where selected reads go: counted, or formatted as SAM lines into a growing buffer. */
typedef struct { int text, json; uint64_t cnt; char* buf; size_t len, cap; int err; } Out;
static void out_put(Out* o, const void* s, size_t n) {
    if (o->len + n > o->cap) { o->cap = (o->len + n) * 2 + 4096; o->buf = realloc(o->buf, o->cap); }
    memcpy(o->buf + o->len, s, n); o->len += n;
}
static void out_str(Out* o, const char* s) { out_put(o, s, strlen(s)); }
static void out_fmt(Out* o, const char* fmt, long long v) { char t[32]; int n = snprintf(t, sizeof t, fmt, v); out_put(o, t, (size_t)n); }
static void out_g(Out* o, float f) { char t[64]; int n = snprintf(t, sizeof t, "%g", (double)f); out_put(o, t, (size_t)n); }
static uint32_t val_size(uint8_t t) { return (t == 'c' || t == 'C') ? 1 : (t == 's' || t == 'S') ? 2 : (t == 'i' || t == 'I' || t == 'f') ? 4 : 0; }
static void out_val(Out* o, uint8_t t, const uint8_t* e) {                /* one integer (signed or unsigned as stored) or float value */
    switch (t) {
        case 'c': out_fmt(o, "%lld", (int8_t)e[0]); break;
        case 'C': out_fmt(o, "%lld", e[0]); break;
        case 's': out_fmt(o, "%lld", (int16_t)(e[0] | (e[1] << 8))); break;
        case 'S': out_fmt(o, "%lld", (uint16_t)(e[0] | (e[1] << 8))); break;
        case 'i': out_fmt(o, "%lld", (int32_t)rd32(e)); break;
        case 'I': out_fmt(o, "%lld", rd32(e)); break;
        default: { uint32_t w = rd32(e); float f; memcpy(&f, &w, 4); out_g(o, f); }
    }
}
static int sam_fail(Out* o, const char* m) { if (!o->err) snprintf(g_err, sizeof g_err, "%s", m); o->err = 1; return -1; }
/* BamRead.toSam (read.d:695-760) of one record, '\n' after it */
static int sam_line(const Bam* b, const Rec* x, Out* o) {
    const uint8_t* p = x->p; const uint32_t bs = x->bs;
    const int32_t ref = (int32_t)rd32(p), pos = (int32_t)rd32(p + 4), l_seq = (int32_t)rd32(p + 16), nref = (int32_t)rd32(p + 20), npos = (int32_t)rd32(p + 24), tlen = (int32_t)rd32(p + 28);
    const uint32_t bmn = rd32(p + 8), fnc = rd32(p + 12), l_name = bmn & 0xFF, mapq = (bmn >> 8) & 0xFF, flag = fnc >> 16, n_cig = fnc & 0xFFFF;
    if (ref < -1 || ref >= b->n_ref) return sam_fail(o, "reference ID out of range");
    if (nref != ref && (nref < -1 || nref >= b->n_ref)) return sam_fail(o, "mate reference ID out of range");
    const uint64_t a0 = 32ull + l_name + 4ull * n_cig + ((uint64_t)(uint32_t)l_seq + 1) / 2 + (uint32_t)l_seq;
    if (l_seq < 0 || a0 > bs) return sam_fail(o, "record fields run past block_size");
    out_put(o, p + 32, l_name ? l_name - 1 : 0);                         /* name */
    out_fmt(o, "\t%lld\t", flag);
    if (ref == -1) out_str(o, "*"); else out_str(o, b->names[ref]);
    out_fmt(o, "\t%lld", (int32_t)((uint32_t)pos + 1u));                  /* position + 1 in D's int: wraps */
    out_fmt(o, "\t%lld\t", mapq);
    const uint8_t* cg = p + 32 + l_name;
    if (!n_cig) out_str(o, "*");
    for (uint32_t i = 0; i < n_cig; i++) { uint32_t c = rd32(cg + 4 * i); out_fmt(o, "%lld", c >> 4); out_put(o, &"MIDNSHP=X???????"[c & 15], 1); }
    out_str(o, "\t");
    if (nref == ref) out_str(o, nref == -1 ? "*\t" : "=\t");
    else if (nref == -1) out_str(o, "*\t");
    else { out_str(o, b->names[nref]); out_str(o, "\t"); }
    out_fmt(o, "%lld\t", (int32_t)((uint32_t)npos + 1u));
    out_fmt(o, "%lld\t", tlen);
    const uint8_t* sq = cg + 4 * n_cig; const uint8_t* qs = sq + ((uint32_t)l_seq + 1) / 2;
    if (l_seq == 0) out_str(o, "*");
    for (int32_t i = 0; i < l_seq; i++) out_put(o, &"=ACMGRSVTWYHKDBN"[(i & 1) ? (sq[i >> 1] & 15) : (sq[i >> 1] >> 4)], 1);
    out_str(o, "\t");
    if (l_seq == 0 || qs[0] == 0xFF) out_str(o, "*");
    else for (int32_t i = 0; i < l_seq; i++) { char c = (char)(uint8_t)(qs[i] + 33); out_put(o, &c, 1); }
    const uint8_t* ax = p + a0; const size_t alen = bs - a0;
    size_t off = 0;
    while (off + 1 < alen) {                                                /* opApply, read.d:1173-1186 */
        out_str(o, "\t"); out_put(o, ax + off, 2); out_str(o, ":");
        off += 2;
        if (off >= alen) return sam_fail(o, "tag runs past the record");
        const uint8_t t = ax[off++];
        const uint32_t sz = val_size(t);
        if (t == 'A') {
            if (off + 1 > alen) return sam_fail(o, "tag runs past the record");
            out_str(o, "A:"); out_put(o, ax + off, 1); off += 1;
        } else if (sz) {                                                    /* c C s S i I: "i:", f: "f:" */
            if (off + sz > alen) return sam_fail(o, "tag runs past the record");
            out_str(o, t == 'f' ? "f:" : "i:"); out_val(o, t, ax + off); off += sz;
        } else if (t == 'Z' || t == 'H') {
            const uint8_t* z = memchr(ax + off, 0, alen - off);
            if (!z) return sam_fail(o, "Z or H value without its NUL");
            out_put(o, &t, 1); out_str(o, ":"); out_put(o, ax + off, (size_t)(z - (ax + off))); off = (size_t)(z - ax) + 1;
        } else if (t == 'B') {
            if (off + 5 > alen) return sam_fail(o, "B array runs past the record");
            const uint8_t et = ax[off]; const uint32_t n = rd32(ax + off + 1), esz = val_size(et); off += 5;
            if (!esz) return sam_fail(o, "unknown B array element type");
            if ((uint64_t)n * esz > alen - off) return sam_fail(o, "B array runs past the record");
            out_str(o, "B:"); out_put(o, &et, 1); out_str(o, ",");
            for (uint32_t i = 0; i < n; i++) { if (i) out_str(o, ","); out_val(o, et, ax + off + (size_t)esz * i); }
            off += (size_t)n * esz;
        } else return sam_fail(o, "unknown tag type");
    }
    out_str(o, "\n");
    return 0;
}

/* ---- BamRead.toJson (read.d:768-830) with BioD's JSON writers (bio/core/utils/format.d) */
static const char specialCharacterTable[256] = {                            /* format.d:221-240: the escape letter, 0 = written as it is */
    ['\b'] = 'b', ['\t'] = 't', ['\n'] = 'n', ['\f'] = 'f', ['\r'] = 'r', ['"'] = '"', ['/'] = '/', ['\\'] = '\\' };
static void writeStringJson(Out* o, const uint8_t* s, size_t n) {          /* format.d:242-254 */
    out_str(o, "\"");
    for (size_t i = 0; i < n; i++) {
        const char sc = specialCharacterTable[s[i]];
        if (sc == 0) out_put(o, s + i, 1);
        else { out_str(o, "\\"); out_put(o, &sc, 1); }
    }
    out_str(o, "\"");
}
/* itoa (format.d:66-87): digits of the magnitude, reversed.  BioD negates a signed value in int before widening it to ulong, so at INT32_MIN it
 * would print -18446744071562067968; this restatement prints -2147483648 as the SAM lines do (a stated deviation, DESIGN.md section 8). */
static void itoa_json(Out* o, long long value) {
    char str[32], *wstr = str;
    unsigned long long uvalue = value < 0 ? (unsigned long long)(-value) : (unsigned long long)value;
    do { *wstr++ = (char)(48 + (uvalue % 10)); } while (uvalue /= 10);
    if (value < 0) *wstr++ = '-';
    for (char *b = str, *e = wstr - 1, t; e > b; b++, e--) { t = *e; *e = *b; *b = t; }
    out_put(o, str, (size_t)(wstr - str));
}
static void writeFloatJson(Out* o, float value) {                            /* format.d:196-212 */
    if (isfinite(value)) out_g(o, value);
    else if (value == INFINITY) out_str(o, "1.0e+1024");
    else if (value == -INFINITY) out_str(o, "-1.0e+1024");
    else out_str(o, "null");
}
static void json_val(Out* o, uint8_t t, const uint8_t* e) {                 /* one integer or float value (tagvalue.d:515-538) */
    switch (t) {
        case 'c': itoa_json(o, (int8_t)e[0]); break;
        case 'C': itoa_json(o, e[0]); break;
        case 's': itoa_json(o, (int16_t)(e[0] | (e[1] << 8))); break;
        case 'S': itoa_json(o, (uint16_t)(e[0] | (e[1] << 8))); break;
        case 'i': itoa_json(o, (int32_t)rd32(e)); break;
        case 'I': itoa_json(o, rd32(e)); break;
        default: { uint32_t w = rd32(e); float f; memcpy(&f, &w, 4); writeFloatJson(o, f); }
    }
}
static int json_line(const Bam* b, const Rec* x, Out* o) {
    const uint8_t* p = x->p; const uint32_t bs = x->bs;
    const int32_t ref = (int32_t)rd32(p), pos = (int32_t)rd32(p + 4), l_seq = (int32_t)rd32(p + 16), nref = (int32_t)rd32(p + 20), npos = (int32_t)rd32(p + 24), tlen = (int32_t)rd32(p + 28);
    const uint32_t bmn = rd32(p + 8), fnc = rd32(p + 12), l_name = bmn & 0xFF, mapq = (bmn >> 8) & 0xFF, flag = fnc >> 16, n_cig = fnc & 0xFFFF;
    if (ref < -1 || ref >= b->n_ref) return sam_fail(o, "reference ID out of range");
    if (nref != ref && (nref < -1 || nref >= b->n_ref)) return sam_fail(o, "mate reference ID out of range");
    const uint64_t a0 = 32ull + l_name + 4ull * n_cig + ((uint64_t)(uint32_t)l_seq + 1) / 2 + (uint32_t)l_seq;
    if (l_seq < 0 || a0 > bs) return sam_fail(o, "record fields run past block_size");
    out_str(o, "{\"qname\":"); writeStringJson(o, p + 32, l_name ? l_name - 1 : 0);
    out_str(o, ",\"flag\":"); itoa_json(o, flag);
    out_str(o, ",\"rname\":");
    if (ref == -1) out_str(o, "\"*\""); else writeStringJson(o, (const uint8_t*)b->names[ref], strlen(b->names[ref]));
    out_str(o, ",\"pos\":"); itoa_json(o, (int32_t)((uint32_t)pos + 1u));        /* position + 1 in D's int: wraps */
    out_str(o, ",\"mapq\":"); itoa_json(o, mapq);
    out_str(o, ",\"cigar\":\"");
    const uint8_t* cg = p + 32 + l_name;
    if (!n_cig) out_str(o, "*");
    for (uint32_t i = 0; i < n_cig; i++) { uint32_t c = rd32(cg + 4 * i); itoa_json(o, c >> 4); out_put(o, &"MIDNSHP=X???????"[c & 15], 1); }
    out_str(o, "\"");
    out_str(o, ",\"rnext\":");
    if (nref == ref) out_str(o, nref == -1 ? "\"*\"" : "\"=\"");
    else if (nref == -1) out_str(o, "\"*\"");
    else writeStringJson(o, (const uint8_t*)b->names[nref], strlen(b->names[nref]));
    out_str(o, ",\"pnext\":"); itoa_json(o, (int32_t)((uint32_t)npos + 1u));
    out_str(o, ",\"tlen\":"); itoa_json(o, tlen);
    out_str(o, ",\"seq\":\"");
    const uint8_t* sq = cg + 4 * n_cig; const uint8_t* qs = sq + ((uint32_t)l_seq + 1) / 2;
    if (l_seq == 0) out_str(o, "*");
    for (int32_t i = 0; i < l_seq; i++) out_put(o, &"=ACMGRSVTWYHKDBN"[(i & 1) ? (sq[i >> 1] & 15) : (sq[i >> 1] >> 4)], 1);
    out_str(o, "\"");
    out_str(o, ",\"qual\":");                                                /* writeArrayJson (format.d:256-270) of the raw bytes */
    if (l_seq == 0) out_str(o, "[]");
    else { out_str(o, "["); for (int32_t i = 0; i < l_seq; i++) { if (i) out_str(o, ","); itoa_json(o, qs[i]); } out_str(o, "]"); }
    out_str(o, ",\"tags\":{");
    const uint8_t* ax = p + a0; const size_t alen = bs - a0;
    size_t off = 0; int not_first = 0;
    while (off + 1 < alen) {                                                /* opApply, read.d:1173-1186 */
        if (not_first) out_str(o, ",");
        writeStringJson(o, ax + off, 2); out_str(o, ":");
        off += 2;
        if (off >= alen) return sam_fail(o, "tag runs past the record");
        const uint8_t t = ax[off++];
        const uint32_t sz = val_size(t);
        if (t == 'A') {
            if (off + 1 > alen) return sam_fail(o, "tag runs past the record");
            writeStringJson(o, ax + off, 1); off += 1;                       /* writeCharJson */
        } else if (sz) {
            if (off + sz > alen) return sam_fail(o, "tag runs past the record");
            json_val(o, t, ax + off); off += sz;
        } else if (t == 'Z' || t == 'H') {
            const uint8_t* z = memchr(ax + off, 0, alen - off);
            if (!z) return sam_fail(o, "Z or H value without its NUL");
            writeStringJson(o, ax + off, (size_t)(z - (ax + off))); off = (size_t)(z - ax) + 1;
        } else if (t == 'B') {
            if (off + 5 > alen) return sam_fail(o, "B array runs past the record");
            const uint8_t et = ax[off]; const uint32_t n = rd32(ax + off + 1), esz = val_size(et); off += 5;
            if (!esz) return sam_fail(o, "unknown B array element type");
            if ((uint64_t)n * esz > alen - off) return sam_fail(o, "B array runs past the record");
            if (n == 0) out_str(o, "[]");
            else {
                out_str(o, "[");
                for (uint32_t i = 0; i + 1 < n; i++) { json_val(o, et, ax + off + (size_t)esz * i); out_str(o, ","); }
                json_val(o, et, ax + off + (size_t)esz * (n - 1)); out_str(o, "]");
            }
            off += (size_t)n * esz;
        } else return sam_fail(o, "unknown tag type");
        not_first = 1;
    }
    out_str(o, "}}\n");
    return 0;
}

static void emit(const Bam* b, const Rec* x, Out* o) {
    if (!o->text) { o->cnt++; return; }
    if (!o->err) (o->json ? json_line : sam_line)(b, x, o);
}

/* ---- isValid (BioD/bio/std/hts/bam/validation/alignment.d:138-562) as BooleanValidator (:528-562) runs it: every onError returns false, so
 * each check stops at its first failure and _visitAlignment (:335-341) stops at the first failing check.  p: the refID field, bs: block_size
 * (the name, CIGAR, sequence and qualities lie inside it: the engine refuses the file otherwise).  Returns 0 (valid), 1 (invalid) or 2 where
 * the tag walk throws or reads past the record (opApply, read.d:1173-1186; readValue, tagvalue.d:468-504), *why saying which. */
typedef struct { const uint8_t* key; uint8_t t; const uint8_t* v; size_t n; } Tag;     /* n: Z / H length without the NUL, B element count */
/* one step of opApply at offset *off of the aux bytes: 0 and the tag, or 2 and *why */
static int tag_next(const uint8_t* ax, size_t alen, size_t* off, Tag* g, const char** why) {
    g->key = ax + *off; *off += 2;
    if (*off >= alen) { *why = "tag runs past the record"; return 2; }
    const uint8_t t = ax[(*off)++]; const uint32_t sz = val_size(t);
    g->t = t; g->v = ax + *off; g->n = 1;
    if (t == 'A') {
        if (*off + 1 > alen) { *why = "tag runs past the record"; return 2; }
        *off += 1;
    } else if (sz) {
        if (*off + sz > alen) { *why = "tag runs past the record"; return 2; }
        *off += sz;
    } else if (t == 'Z' || t == 'H') {
        const uint8_t* z = memchr(ax + *off, 0, alen - *off);
        if (!z) { *why = "Z or H value without its NUL"; return 2; }
        g->n = (size_t)(z - (ax + *off)); *off = (size_t)(z - ax) + 1;
    } else if (t == 'B') {
        if (*off + 5 > alen) { *why = "B array runs past the record"; return 2; }
        const uint32_t n = rd32(ax + *off + 1), esz = val_size(ax[*off]); *off += 5;
        if (!esz) { *why = "unknown B array element type"; return 2; }
        if ((uint64_t)n * esz > alen - *off) { *why = "B array runs past the record"; return 2; }
        g->n = n; *off += (size_t)n * esz;
    } else { *why = "unknown tag type"; return 2; }
    return 0;
}
static int is_integer(uint8_t t) { return t == 'c' || t == 'C' || t == 's' || t == 'S' || t == 'i' || t == 'I'; }
static int key_in(const uint8_t* k, const char* list) {      /* list: keys separated by one space */
    for (size_t i = 0; i + 1 < strlen(list); i += 3) if (k[0] == (uint8_t)list[i] && k[1] == (uint8_t)list[i + 1]) return 1;
    return 0;
}
/* checkTagValue (:428-526) of a predefined key (PredefinedTags, :83-119); other keys pass (additionalChecksIfTheTagIsPredefined, :407-426) */
static int check_tag_value(const Tag* g, int32_t l_seq) {
    const uint8_t* k = g->key;
    if (key_in(k, "AM AS CM CP FI H0 H1 H2 HI IH MQ NH NM OP PQ SM TC UQ")) return is_integer(g->t);      /* 1. type: int */
    if (key_in(k, "FZ")) return g->t == 'B' && g->v[0] == 'S';                                          /*    ushort[] */
    if (!key_in(k, "BC BQ CC CQ CS E2 FS LB MD OQ OC PG PU Q2 R2 RG U2")) return 1;
    if (g->t != 'Z') return 0;                                                /*    string: is_string, and not 'H' */
    const uint8_t* s = g->v; const size_t n = g->n;
    if (key_in(k, "CQ E2 OQ Q2 U2")) {                                        /* 2. "*" or all [!-~] */
        int all = 1; for (size_t i = 0; i < n; i++) if (!(s[i] >= '!' && s[i] <= '~')) all = 0;
        if (!(n == 1 && s[0] == '*') && !all) return 0;
    }
    if (key_in(k, "BQ E2") && n != (size_t)l_seq) return 0;                  /* 3. the sequence's length */
    if (key_in(k, "MD")) {                                                    /* 4. the scanner of :483-523 */
        int valid = 1;
        if (n == 0) valid = 0;
        if (!isdigit(s[0])) valid = 0;
        size_t i = 1;
        while (i < n && isdigit(s[i])) ++i;
        while (i < n) {
            if (isupper(s[i])) ++i;
            else if (s[i] == '^') {
                ++i;
                if (i == n || !isupper(s[i])) { valid = 0; break; }
                while (i < n && isupper(s[i])) ++i;
            } else { valid = 0; break; }
            if (i == n || !isdigit(s[i])) { valid = 0; break; }
            while (i < n && isdigit(s[i])) ++i;
        }
        if (i < n) valid = 0;
        if (!valid) return 0;
    }
    return 1;
}
/* isValid(key, value, al) (:343-405): the value's own type, then the predefined keys */
static int tag_is_valid(const Tag* g, int32_t l_seq) {
    if (g->t == 'H') {
        if (g->n == 0) return 0;
        for (size_t i = 0; i < g->n; i++) if (!isxdigit(g->v[i])) return 0;
    } else if (g->t == 'A') {
        if (!(g->v[0] >= '!' && g->v[0] <= '~')) return 0;
    } else if (g->t == 'Z') {
        if (g->n == 0) return 0;
        for (size_t i = 0; i < g->n; i++) if (!(g->v[i] >= ' ' && g->v[i] <= '~')) return 0;
    }
    return check_tag_value(g, l_seq);
}
static int alignment_valid(const uint8_t* p, uint32_t bs, const char** why) {
    const int32_t pos = (int32_t)rd32(p + 4), l_seq = (int32_t)rd32(p + 16);
    const uint32_t l_name = p[8], n_cig = rd32(p + 12) & 0xFFFF;
    /* invalidReadName (:170-190): name = the first l_read_name - 1 bytes; l_read_name 0 slices [32 .. 31], whose length wraps */
    const size_t name_len = (size_t)l_name - 1;
    if (name_len == 0) return 1;
    if (name_len > 255) return 1;
    for (size_t i = 0; i < name_len; i++) { const uint8_t c = p[32 + i]; if (c < '!' || c > '~' || c == '@') return 1; }
    /* invalidPosition (:192-200) */
    if (pos < -1 || pos > ((1 << 29) - 2)) return 1;
    /* invalidQualityData (:202-212) */
    const uint8_t* cg = p + 32 + l_name;
    const uint8_t* qs = cg + 4 * n_cig + ((uint32_t)l_seq + 1) / 2;
    int all_ff = 1, all_ok = 1;
    for (int32_t i = 0; i < l_seq; i++) { if (qs[i] != 0xFF) all_ff = 0; if (qs[i] > 93) all_ok = 0; }
    if (!all_ff && !all_ok) return 1;
    /* invalidCigar (:214-268): op types "MIDNSHP=X????????"[op & 15] (cigar.d:110) */
    if (n_cig) {
        char ty[65536];
        for (uint32_t i = 0; i < n_cig; i++) ty[i] = "MIDNSHP=X????????"[rd32(cg + 4 * i) & 15];
        if (n_cig > 2) for (uint32_t i = 1; i + 1 < n_cig; i++) if (ty[i] == 'H') return 1;       /* internalHardClipping */
        if (n_cig > 2) {                                                                             /* internalSoftClipping */
            uint32_t a = 0, e = n_cig;
            if (ty[a] == 'H') a++;
            if (ty[e - 1] == 'H') e--;
            if (e - a > 2) for (uint32_t i = a + 1; i + 1 < e; i++) if (ty[i] == 'S') return 1;
        }
        int32_t sum = 0;                                                                             /* inconsistentLength: reduce in int, wrapping */
        for (uint32_t i = 0; i < n_cig; i++) if (strchr("MIS=X", ty[i])) sum = (int32_t)((uint32_t)sum + (rd32(cg + 4 * i) >> 4));
        if (l_seq > 0 && l_seq != sum) return 1;
    }
    /* invalidTags (:272-333): every tag is visited (someTagIsBad's return leaves only that nested function) */
    const uint32_t a0 = 32 + l_name + 4 * n_cig + ((uint32_t)l_seq + 1) / 2 + (uint32_t)l_seq;
    const uint8_t* ax = p + a0; const size_t alen = bs - a0;
    int all_tags_are_good = 1, all_distinct = 1;
    uint16_t keys[256]; size_t i = 0;
    for (size_t off = 0; off + 1 < alen;) {
        Tag g;
        if (tag_next(ax, alen, &off, &g, why)) return 2;
        if (!tag_is_valid(&g, l_seq)) all_tags_are_good = 0;
        const uint16_t k = (uint16_t)(g.key[0] | (g.key[1] << 8));
        if (i < 256) {
            keys[i] = k;
            if (all_distinct) for (size_t j = 0; j < i; ++j) if (keys[i] == keys[j]) { all_distinct = 0; break; }
            i += 1;
        } else if (all_distinct) {                                             /* must be exactly one: count this key over all the tags */
            int found = 0;
            for (size_t o2 = 0; o2 + 1 < alen;) {
                Tag g2;
                if (tag_next(ax, alen, &o2, &g2, why)) return 2;
                if ((uint16_t)(g2.key[0] | (g2.key[1] << 8)) == k) { if (found == 1) { all_distinct = 0; break; } ++found; }
            }
        }
    }
    return (all_tags_are_good && all_distinct) ? 0 : 1;
}
/* The validator alone on one record (p: its refID field): 0 valid, 1 invalid, 2 refused (view_count_oracle_error() says why). */
int view_valid_oracle(const uint8_t* p, uint32_t bs) {
    const char* why = NULL; g_err[0] = 0;
    const int v = alignment_valid(p, bs, &why);
    if (v == 2) snprintf(g_err, sizeof g_err, "%s", why);
    return v;
}
static int g_valid;
/* -v for the calls that follow (the existing entry points keep their signatures) */
void view_count_oracle_set_valid(int on) { g_valid = on != 0; }

/* The filter chain of view_main (view.d:265-289): SubsampleFilter in front, then NullFilter, ValidAlignmentFilter (-v), FlagBitFilter; -F comes
 * after them (the tests apply it to the file).  A record the validator would abort on stops the run (o's error). */
static int keep_read(const Rec* x, unsigned fs, unsigned fu, int sub, uint64_t thr, uint64_t seed, Out* o) {
    if (sub && (view_count_oracle_hash(x->name, x->l_name ? x->l_name - 1 : 0, seed) & 0xFFFFFFFFull) >= thr) return 0;
    if (g_valid) {
        const char* why = NULL; const int v = alignment_valid(x->p, x->bs, &why);
        if (v == 2) { sam_fail(o, why); return 0; }
        if (v) return 0;
    }
    if ((x->flag & fs) != fs || (x->flag & fu)) return 0;
    return 1;
}
/* BamReadFilter (randomaccessmanager.d:366-462): number of records of rec[0..n) the state machine yields for the sorted, non-overlapping regions. */
static void read_filter_walk(const Bam* b, const Reg* regs, size_t nreg, size_t i0, unsigned fs, unsigned fu, int sub, uint64_t thr, uint64_t seed, Out* out) {
    size_t ri = 0; const uint32_t ref_id = regs[0].ref;
    for (size_t i = i0; i < b->nr && ri < nreg;) {
        const Rec* x = &b->r[i];
        uint32_t cur = (uint32_t)x->ref;                          /* cast(uint)ref_id */
        if (cur > ref_id) break;
        if (cur < ref_id) { i++; continue; }
        if ((uint32_t)x->pos >= regs[ri].end) { ri++; continue; }  /* int position against uint end: as unsigned */
        int yield;
        if ((uint32_t)x->pos > regs[ri].start) yield = 1;
        else if ((int64_t)(int32_t)x->pos + x->bc <= (int64_t)regs[ri].start) yield = 0;
        else yield = 1;
        if (yield && keep_read(x, fs, fu, sub, thr, seed, out)) emit(b, x, out);
        i++;
    }
}

static int cmp_reg(const void* a, const void* b) {
    const Reg *x = a, *y = b;
    if (x->ref != y->ref) return x->ref < y->ref ? -1 : 1;
    if (x->start != y->start) return x->start < y->start ? -1 : 1;
    return x->end < y->end ? -1 : x->end > y->end;
}

/* mode 0: every record; 1: -L regions (as parseBed hands them over: any order, merged here as nonOverlappingIntervals does, bed.d:43-58);
 * 2: positional regions (ref, start, end) in the given order, a ref of 0xFFFFFFFF being '*' in its place, plus n_star '*' queries at the end.
 * Returns 0 or -1 (view_count_oracle_error()). */
static int view_stream(const Bam* b, unsigned flag_set, unsigned flag_unset, int subsample, uint64_t threshold, uint64_t seed,
                       int mode, const uint32_t* regs, size_t nreg, unsigned n_star, Out* out) {
    int rc = 0;
    if (mode == 0) {
        for (size_t i = 0; i < b->nr; i++) if (keep_read(&b->r[i], flag_set, flag_unset, subsample, threshold, seed, out)) emit(b, &b->r[i], out);
    } else if (mode == 1) {
        Reg* r = malloc((nreg + 1) * sizeof(Reg)); size_t m = 0;
        for (size_t i = 0; i < nreg; i++) if (regs[3 * i + 1] < regs[3 * i + 2]) { r[m].ref = regs[3 * i]; r[m].start = regs[3 * i + 1]; r[m].end = regs[3 * i + 2]; m++; }
        qsort(r, m, sizeof(Reg), cmp_reg);
        size_t k = 0;
        for (size_t i = 0; i < m; i++) { if (k && r[k - 1].ref == r[i].ref && r[k - 1].end >= r[i].start) { if (r[i].end > r[k - 1].end) r[k - 1].end = r[i].end; } else r[k++] = r[i]; }
        m = k;
        if (b->sorted) {                                   /* getReadsOverlapping: one BamReadFilter per reference group, joined */
            for (size_t g = 0; g < m;) { size_t e = g; while (e < m && r[e].ref == r[g].ref) e++; read_filter_walk(b, r + g, e - g, 0, flag_set, flag_unset, subsample, threshold, seed, out); g = e; }
        } else if (!m) {
            snprintf(g_err, sizeof g_err, "-L on an unsorted file with no region on the file's references: BedFilter indexes an empty list"); rc = -1;
        } else {                                           /* BedFilter: trees_.length = bed.back.ref_id + 1 */
            const uint32_t ntrees = r[m - 1].ref + 1;
            for (size_t i = 0; i < b->nr; i++) {
                const Rec* x = &b->r[i];
                if (!keep_read(x, flag_set, flag_unset, subsample, threshold, seed, out)) continue;      /* the chain, then BedFilter */
                if (x->ref < 0 || (uint32_t)x->ref >= ntrees) continue;
                const uint32_t s = (uint32_t)x->pos, t = (uint32_t)((int32_t)x->pos + (int32_t)x->bc);
                for (size_t j = 0; j < m; j++) if (r[j].ref == (uint32_t)x->ref && r[j].end > s && r[j].start < t) { emit(b, x, out); break; }
            }
        }
        free(r);
    } else {
        for (size_t i = 0; i < nreg && !rc; i++) {
            Reg one = {regs[3 * i], regs[3 * i + 1], regs[3 * i + 2]};
            if (one.ref == 0xFFFFFFFFu) continue;
            if (!(one.start < one.end)) { snprintf(g_err, sizeof g_err, "start must be less than end"); rc = -1; }
        }
        for (size_t i = 0; i < nreg && !rc; i++) {
            Reg one = {regs[3 * i], regs[3 * i + 1], regs[3 * i + 2]};
            if (one.ref != 0xFFFFFFFFu) { read_filter_walk(b, &one, 1, 0, flag_set, flag_unset, subsample, threshold, seed, out); continue; }
            /* '*' in its place: unmappedReads, the first refID -1 record, then everything to EOF */
            size_t k = 0; while (k < b->nr && b->r[k].ref != -1) k++;
            for (; k < b->nr; k++) if (keep_read(&b->r[k], flag_set, flag_unset, subsample, threshold, seed, out)) emit(b, &b->r[k], out);
        }
        for (unsigned k = 0; k < n_star && !rc; k++) {     /* unmappedReads: the first refID -1 record, then everything to EOF */
            size_t i = 0; while (i < b->nr && b->r[i].ref != -1) i++;
            for (; i < b->nr; i++) if (keep_read(&b->r[i], flag_set, flag_unset, subsample, threshold, seed, out)) emit(b, &b->r[i], out);
        }
    }
    if (!rc && out->err) rc = -1;
    return rc;
}

int view_count_oracle(const char* path, unsigned flag_set, unsigned flag_unset, int subsample, uint64_t threshold, uint64_t seed,
                      int mode, const uint32_t* regs, size_t nreg, unsigned n_star, uint64_t* out) {
    Bam b; g_err[0] = 0;
    if (bam_load(path, &b)) { bam_free(&b); return -1; }
    Out o = {0};
    const int rc = view_stream(&b, flag_set, flag_unset, subsample, threshold, seed, mode, regs, nreg, n_star, &o);
    bam_free(&b);
    if (!rc) *out = o.cnt;
    return rc;
}

static int text_oracle(const char* path, unsigned flag_set, unsigned flag_unset, int subsample, uint64_t threshold, uint64_t seed,
                       int mode, const uint32_t* regs, size_t nreg, int json, char** text, size_t* len) {
    Bam b; g_err[0] = 0;
    if (bam_load(path, &b)) { bam_free(&b); return -1; }
    Out o = {0}; o.text = 1; o.json = json;
    const int rc = view_stream(&b, flag_set, flag_unset, subsample, threshold, seed, mode, regs, nreg, 0, &o);
    bam_free(&b);
    if (rc) { free(o.buf); return -1; }
    *text = o.buf; *len = o.len;
    return 0;
}
/* The SAM lines `sambamba view` prints after the header, in the order of its joined stream; *text is freed with view_text_oracle_free(). */
int view_text_oracle(const char* path, unsigned flag_set, unsigned flag_unset, int subsample, uint64_t threshold, uint64_t seed,
                     int mode, const uint32_t* regs, size_t nreg, char** text, size_t* len) {
    return text_oracle(path, flag_set, flag_unset, subsample, threshold, seed, mode, regs, nreg, 0, text, len);
}
/* The records `sambamba view -f json` prints, in the same order; *text is freed with view_text_oracle_free(). */
int view_json_oracle(const char* path, unsigned flag_set, unsigned flag_unset, int subsample, uint64_t threshold, uint64_t seed,
                     int mode, const uint32_t* regs, size_t nreg, char** text, size_t* len) {
    return text_oracle(path, flag_set, flag_unset, subsample, threshold, seed, mode, regs, nreg, 1, text, len);
}
void view_text_oracle_free(char* text) { free(text); }

#ifdef ORACLE_MAIN
static int die(const char* m) { fprintf(stderr, "sambamba-view: %s\n", m); return 1; }
static int conv_u(const char* s, unsigned long long maxv, const char* type, unsigned long long* v) {
    char m[256];
    if (!*s) { snprintf(m, sizeof m, "Unexpected end of input when converting from type string to type %s", type); return die(m); }
    unsigned long long x = 0;
    for (const char* p = s; *p; p++) {
        if (*p < '0' || *p > '9') { snprintf(m, sizeof m, "Unexpected '%c' when converting from type string to type %s", *p, type); return die(m); }
        if (x > (maxv - (unsigned)(*p - '0')) / 10) return die("Conversion positive overflow");
        x = x * 10 + (unsigned)(*p - '0');
    }
    *v = x; return 0;
}
/* region.rl: ref[:beg[-end]], 1-based closed -> 0-based half-open */
static void parse_region(const char* s, char* ref, size_t cap, uint32_t* beg, uint32_t* end) {
    *beg = 0; *end = UINT32_MAX; size_t n = strlen(s), c = (size_t)-1;
    for (size_t t = 0; t < n; t++) if (s[t] == ':') {
        size_t q = t + 1; int ok = q < n && isdigit((unsigned char)s[q]);
        while (q < n && (isdigit((unsigned char)s[q]) || s[q] == ',')) q++;
        if (ok && q < n && s[q] == '-') { q++; if (!(q < n && isdigit((unsigned char)s[q]))) ok = 0; while (q < n && (isdigit((unsigned char)s[q]) || s[q] == ',')) q++; }
        if (ok && q == n) { c = t; break; }
    }
    if (c == (size_t)-1) { snprintf(ref, cap, "%s", s); return; }
    snprintf(ref, cap, "%.*s", (int)c, s);
    long v = 0; size_t q = c + 1;
    while (q < n && s[q] != '-') { if (s[q] != ',') v = v * 10 + (s[q] - '0'); q++; }
    *beg = (uint32_t)(v - 1);
    if (q < n && s[q] == '-') { q++; v = 0; while (q < n) { if (s[q] != ',') v = v * 10 + (s[q] - '0'); q++; } *end = (uint32_t)v; }
}
int main(int argc, char** argv) {
    if (argc < 2 || strcmp(argv[1], "view")) { fprintf(stderr, "usage: view_count_oracle view [-c] [options] in.bam [region ...]\n"); return 1; }
    unsigned long long fs = 0, fu = 0, seed = 0; double frac = NAN; const char* bed = NULL; int count = 0, json = 0;
    const char* pos_args[4096]; int npos = 0;
    for (int i = 2; i < argc; i++) {
        const char* a = argv[i];
        if (!strcmp(a, "-c")) count = 1;
        else if (!strcmp(a, "-v")) g_valid = 1;
        else if (!strncmp(a, "--num-filter=", 13)) {
            char buf[256]; snprintf(buf, sizeof buf, "%s", a + 13); char* sl = strchr(buf, '/');
            if (sl) *sl = 0;
            if (*buf && conv_u(buf, 0xFFFF, "ushort", &fs)) return 1;
            if (sl && sl[1] && conv_u(sl + 1, 0xFFFF, "ushort", &fu)) return 1;
        } else if (!strcmp(a, "-s") && i + 1 < argc) frac = strtod(argv[++i], NULL);
        else if (!strncmp(a, "--subsampling-seed=", 19)) { if (conv_u(a + 19, 0xFFFFFFFFFFFFFFF0ull, "ulong", &seed)) return 1; }
        else if (!strcmp(a, "-L") && i + 1 < argc) bed = argv[++i];
        else if (!strcmp(a, "-f") && i + 1 < argc) {
            const char* f = argv[++i];
            if (strcmp(f, "sam") && strcmp(f, "json")) return die("output format must be sam or json here");
            json = !strcmp(f, "json");
        }
        else if (npos < 4096) pos_args[npos++] = a;
    }
    if (npos < 1) { fprintf(stderr, "usage: view_count_oracle view [-c] [options] in.bam [region ...]\n"); return 1; }
    int sub = !isnan(frac); uint64_t thr = 0;
    if (sub) { double t = 4294967296.0 * frac; if (!(t >= 0)) return die("Conversion negative overflow"); if (t > 18446744073709551616.0) return die("Conversion positive overflow"); thr = t >= 18446744073709551616.0 ? UINT64_MAX : (uint64_t)t; }
    if (bed && npos > 1) return die("specifying both region and BED filename is disallowed");
    Bam b;
    if (bam_load(pos_args[0], &b)) { bam_free(&b); return die(g_err); }
    size_t cap = 1024, n = 0; uint32_t* regs = malloc(cap * 3 * sizeof(uint32_t)); unsigned n_star = 0;
    int mode = 0;
    if (bed) {                                             /* readIntervals (bed.d:59-97): whitespace fields, to!long, beg == end -> end + 1, beg < end kept */
        mode = 1;
        FILE* f = fopen(bed, "rb"); char msg[600];
        if (!f) { snprintf(msg, sizeof msg, "%s: %s", bed, strerror(errno)); bam_free(&b); return die(msg); }
        char line[65536];
        while (fgets(line, sizeof line, f)) {
            char* fld[3]; int nf = 0; char* sv = NULL;
            for (char* t = strtok_r(line, " \t\r\n\v\f", &sv); t && nf < 3; t = strtok_r(NULL, " \t\r\n\v\f", &sv)) fld[nf++] = t;
            if (nf < 2) continue;
            long beg = strtol(fld[1], NULL, 10), end = nf >= 3 ? strtol(fld[2], NULL, 10) : beg + 1;
            if (beg == end) end = beg + 1;
            if (beg >= end) continue;
            int id = -1; for (int r = 0; r < b.n_ref; r++) if (!strcmp(b.names[r], fld[0])) id = r;
            if (id < 0) continue;
            if (n == cap) { cap *= 2; regs = realloc(regs, cap * 3 * sizeof(uint32_t)); }
            regs[3 * n] = (uint32_t)id; regs[3 * n + 1] = (uint32_t)beg; regs[3 * n + 2] = (uint32_t)end; n++;
        }
        fclose(f);
    } else if (npos > 1) {
        mode = 2;
        for (int i = 1; i < npos; i++) {
            if (!strcmp(pos_args[i], "*")) {               /* counted at the end; the text keeps it in its place */
                if (count) { n_star++; continue; }
                if (n == cap) { cap *= 2; regs = realloc(regs, cap * 3 * sizeof(uint32_t)); }
                regs[3 * n] = 0xFFFFFFFFu; regs[3 * n + 1] = 0; regs[3 * n + 2] = 0; n++; continue;
            }
            char ref[4096]; uint32_t beg, end; parse_region(pos_args[i], ref, sizeof ref, &beg, &end);
            int id = -1; for (int r = 0; r < b.n_ref; r++) if (!strcmp(b.names[r], ref)) id = r;
            if (id < 0) { char msg[4200]; snprintf(msg, sizeof msg, "Reference with name %s does not exist", ref); bam_free(&b); return die(msg); }
            if (end == UINT32_MAX) {           /* the reference's length from the binary header */
                size_t o = 8 + rd32(b.u + 4) + 4;
                for (int r = 0; r < id; r++) o += 8 + rd32(b.u + o);
                end = rd32(b.u + o + 4 + rd32(b.u + o));
            }
            if (!(beg < end)) { bam_free(&b); return die("start must be less than end"); }
            if (n == cap) { cap *= 2; regs = realloc(regs, cap * 3 * sizeof(uint32_t)); }
            regs[3 * n] = (uint32_t)id; regs[3 * n + 1] = beg; regs[3 * n + 2] = end; n++;
        }
    }
    bam_free(&b);
    if (!count) {
        if (mode == 2 && !n) mode = 0;
        char* text = NULL; size_t len = 0;
        if (text_oracle(pos_args[0], (unsigned)fs, (unsigned)fu, sub, thr, seed, mode, regs, n, json, &text, &len)) { free(regs); return die(g_err); }
        fwrite(text, 1, len, stdout); free(text); free(regs);
        return 0;
    }
    uint64_t cnt = 0;
    if (view_count_oracle(pos_args[0], (unsigned)fs, (unsigned)fu, sub, thr, seed, mode, regs, n, n_star, &cnt)) { free(regs); return die(g_err); }
    free(regs);
    printf("%llu\n", (unsigned long long)cnt);
    return 0;
}
#endif
