/*
 * flagstat_oracle.c -- CPU restatement of `sambamba flagstat` (TEST INFRASTRUCTURE: the checker of bdepth_run_flagstat and of the
 * CLI's `flagstat` subcommand; nothing of the product links or reads it).
 *
 * Its own record walk over its own zlib inflate, independent of the GPU engine:
 *   BGZF members are framed from their headers (BSIZE of the BC subfield) and inflated with zlib, several threads each taking
 *   whole members into their place in one buffer; the BAM header is skipped and the records are walked in file order the way
 *   BioD's readrange.d:118-173 reads them: fewer than 4 bytes left end the stream quietly, a record cut by the end of the file
 *   is "not enough data in stream".
 *   computeFlagStatistics (sambamba/flagstat.d:31-57) is restated line by line in count_record() below.
 *
 * Library:  int oracle_flagstat(const char* path, uint64_t out[26]);  out[2 * category + qc_failed], categories in the order of
 *           bdepth_flagstat (include/bdepth.h).  0, or -1 with oracle_flagstat_error().
 * CLI:      flagstat_oracle flagstat [-b] in.bam   prints what flagstat_main prints (flagstat.d:131-143).
 */
#define _GNU_SOURCE
#include <fcntl.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

enum { TOTAL, SECONDARY, SUPPLEMENTARY, DUPLICATES, MAPPED, PAIRED, READ1, READ2, PROPER_PAIR, BOTH_MAPPED, SINGLETONS, MATE_DIFF_CHR, MATE_DIFF_CHR_MAPQ5, N_CAT };

static __thread char g_err[512];
const char* oracle_flagstat_error(void) { return g_err; }
static int err(const char* fmt, const char* a) { snprintf(g_err, sizeof g_err, fmt, a); return -1; }

static uint32_t rd16(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8; }
static uint32_t rd32(const uint8_t* p) { return rd16(p) | rd16(p + 2) << 16; }

/* flagstat.d:31-57 for one record.  fnc = flag << 16 | n_cigar_op, bmn = bin << 16 | MAPQ << 8 | l_read_name (SAM spec 4.2). */
static void count_record(uint64_t* out, int32_t ref_id, uint32_t bmn, uint32_t fnc, int32_t mate_ref_id) {
    const uint32_t flag = fnc >> 16, mapq = (bmn >> 8) & 0xFF;
    const int failed = (flag & 0x200) ? 1 : 0;                     /* :33  read.failed_quality_control (read.d:182) */
    const int unmapped = (flag & 0x4) != 0, mate_unmapped = (flag & 0x8) != 0;
    out[2 * TOTAL + failed]++;                                     /* :34  ++reads */
    if (!unmapped) out[2 * MAPPED + failed]++;                     /* :35 */
    if (flag & 0x400) out[2 * DUPLICATES + failed]++;              /* :36  is_duplicate */
    if (flag & 0x100) {                                            /* :37  is_secondary_alignment */
        out[2 * SECONDARY + failed]++;
    } else if (flag & 0x800) {                                     /* :39  is_supplementary */
        out[2 * SUPPLEMENTARY + failed]++;
    } else if (flag & 0x1) {                                       /* :41  is_paired */
        out[2 * PAIRED + failed]++;                                /* :42  ++pair_all */
        if ((flag & 0x2) && !unmapped) out[2 * PROPER_PAIR + failed]++;        /* :43  proper_pair */
        if (flag & 0x40) out[2 * READ1 + failed]++;                /* :44  is_first_of_pair */
        if (flag & 0x80) out[2 * READ2 + failed]++;                /* :45  is_second_of_pair */
        if (mate_unmapped && !unmapped) out[2 * SINGLETONS + failed]++;        /* :46 */
        if (!unmapped && !mate_unmapped) {                         /* :47 */
            out[2 * BOTH_MAPPED + failed]++;                       /* :48  ++pair_map */
            if (ref_id != mate_ref_id) {                           /* :49  ref_id / mate_ref_id as written (read.d:86, :117) */
                out[2 * MATE_DIFF_CHR + failed]++;
                if (mapq >= 5) out[2 * MATE_DIFF_CHR_MAPQ5 + failed]++;       /* :51 */
            }
        }
    }
}

typedef struct { uint64_t coff, cdata, csize, uoff, isize; } Member;
typedef struct { const uint8_t* file; const Member* m; size_t lo, hi; uint8_t* u; int bad; size_t bad_at; } Job;

static void* inflate_job(void* arg) {
    Job* j = (Job*)arg;
    for (size_t i = j->lo; i < j->hi && !j->bad; i++) {
        const Member* m = &j->m[i];
        z_stream z; memset(&z, 0, sizeof z);
        if (inflateInit2(&z, -15) != Z_OK) { j->bad = 1; j->bad_at = i; break; }
        z.next_in = (Bytef*)(j->file + m->cdata); z.avail_in = (uInt)m->csize;
        z.next_out = j->u + m->uoff; z.avail_out = (uInt)m->isize;
        const int rc = inflate(&z, Z_FINISH);
        if (rc != Z_STREAM_END || z.total_out != m->isize) { j->bad = 1; j->bad_at = i; }
        inflateEnd(&z);
    }
    return NULL;
}

int oracle_flagstat(const char* path, uint64_t* out) {
    memset(out, 0, 2 * N_CAT * sizeof(uint64_t));
    const int fd = open(path, O_RDONLY);
    if (fd < 0) return err("Cannot open file `%s' in mode `rb' (No such file or directory)", path);
    struct stat sb;
    if (fstat(fd, &sb) != 0 || sb.st_size == 0) { close(fd); return err("cannot read `%s' or the file is empty", path); }
    const size_t flen = (size_t)sb.st_size;
    const uint8_t* f = (const uint8_t*)mmap(NULL, flen, PROT_READ, MAP_PRIVATE, fd, 0);
    close(fd);
    if (f == MAP_FAILED) return err("cannot mmap `%s'", path);
    /* frame the BGZF members */
    size_t cap = 1024, n = 0, off = 0; uint64_t total_u = 0; int rc = 0;
    Member* ms = (Member*)malloc(cap * sizeof(Member));
    while (off < flen) {
        if (off + 18 > flen || f[off] != 31 || f[off + 1] != 139 || f[off + 2] != 8 || !(f[off + 3] & 4)) { rc = err("%s: not a BGZF member (or a truncated one)", path); goto done; }
        const size_t xlen = rd16(f + off + 10); size_t bsize = 0;
        for (size_t x = off + 12; x + 4 <= off + 12 + xlen && x + 4 <= flen; x += 4 + rd16(f + x + 2))
            if (f[x] == 'B' && f[x + 1] == 'C' && rd16(f + x + 2) == 2 && x + 6 <= flen) bsize = rd16(f + x + 4) + 1;
        if (!bsize || off + bsize > flen || bsize < 12 + xlen + 8) { rc = err("%s: BGZF member without a usable BSIZE (or cut by the end of the file)", path); goto done; }
        if (n == cap) { cap *= 2; ms = (Member*)realloc(ms, cap * sizeof(Member)); }
        const uint64_t isize = rd32(f + off + bsize - 4);
        ms[n++] = (Member){off, off + 12 + xlen, bsize - 12 - xlen - 8, total_u, isize};
        total_u += isize; off += bsize;
    }
    {
        uint8_t* u = (uint8_t*)malloc(total_u + 1);
        if (!u) { rc = err("%s: out of memory for the inflated stream", path); goto done; }
        long nt = sysconf(_SC_NPROCESSORS_ONLN); if (nt < 1) nt = 1; if (nt > 32) nt = 32; if ((size_t)nt > n) nt = n ? (long)n : 1;
        Job jobs[32]; pthread_t th[32];
        for (long t = 0; t < nt; t++) { jobs[t] = (Job){f, ms, n * t / nt, n * (t + 1) / nt, u, 0, 0}; pthread_create(&th[t], NULL, inflate_job, &jobs[t]); }
        for (long t = 0; t < nt; t++) pthread_join(th[t], NULL);
        for (long t = 0; t < nt; t++) if (jobs[t].bad) { char at[64]; snprintf(at, sizeof at, "%llu", (unsigned long long)ms[jobs[t].bad_at].coff); free(u); rc = err("DEFLATE error in the BGZF member at offset %s", at); goto done; }
        /* header: magic, l_text, text, n_ref, (l_name, name, l_ref) x n_ref */
        uint64_t o = 0;
        if (total_u < 12 || memcmp(u, "BAM\1", 4) != 0) { free(u); rc = err("%s: Invalid file format: expected BAM\\1", path); goto done; }
        o = 8 + (uint64_t)rd32(u + 4);
        if (o + 4 > total_u) { free(u); rc = err("%s: truncated BAM header", path); goto done; }
        const uint32_t n_ref = rd32(u + o); o += 4;
        for (uint32_t r = 0; r < n_ref; r++) {
            if (o + 4 > total_u || o + 8 + rd32(u + o) > total_u) { free(u); rc = err("%s: truncated BAM header", path); goto done; }
            o += 8 + rd32(u + o);
        }
        /* records (readrange.d:118-173) */
        while (o + 4 <= total_u) {
            const uint32_t bs = rd32(u + o);
            if (bs < 32) { free(u); rc = err("%s: corrupt BAM record (block_size < 32)", path); goto done; }
            if (o + 4 + bs > total_u) { free(u); rc = err("not enough data in stream%s", ""); goto done; }
            const uint8_t* p = u + o + 4;
            count_record(out, (int32_t)rd32(p), rd32(p + 8), rd32(p + 12), (int32_t)rd32(p + 20));
            o += 4 + (uint64_t)bs;
        }
        free(u);
    }
done:
    free(ms);
    munmap((void*)f, flen);
    return rc;
}

#ifdef ORACLE_MAIN
/* percent (flagstat.d:66): to!float(a) / b * 100.0 -- a float quotient, multiplied in double (100.0 is a double literal), returned as
 * float; printed with "%.2f%%" (:70), taken to equal printf's %.2f of the float widened to double. */
static void percent_str(char* t, size_t n, uint64_t a, uint64_t b) {
    if (b == 0) { snprintf(t, n, "N/A"); return; }
    const float p = (float)((double)((float)a / (float)b) * 100.0);
    snprintf(t, n, "%.2f%%", (double)p);
}

static void param(const char* d, const uint64_t* p, int tab) {
    if (tab) printf("%s,%llu,%llu\n", d, (unsigned long long)p[0], (unsigned long long)p[1]);
    else printf("%llu + %llu %s\n", (unsigned long long)p[0], (unsigned long long)p[1], d);
}
static void param_pct(const char* d, const uint64_t* p, const uint64_t* t, int tab) {
    char a0[64], a1[64]; percent_str(a0, sizeof a0, p[0], t[0]); percent_str(a1, sizeof a1, p[1], t[1]);
    if (tab) printf("%s,%llu:%s,%llu:%s\n", d, (unsigned long long)p[0], a0, (unsigned long long)p[1], a1);
    else printf("%llu + %llu %s (%s:%s)\n", (unsigned long long)p[0], (unsigned long long)p[1], d, a0, a1);
}
int main(int argc, char** argv) {
    int tab = 0; const char* in = NULL;
    if (argc < 2 || strcmp(argv[1], "flagstat") != 0) { fprintf(stderr, "usage: flagstat_oracle flagstat [-b] in.bam\n"); return 1; }
    for (int i = 2; i < argc; i++) { if (!strcmp(argv[i], "-b") || !strcmp(argv[i], "--tabular")) tab = 1; else if (!in) in = argv[i]; }
    if (!in) { fprintf(stderr, "usage: flagstat_oracle flagstat [-b] in.bam\n"); return 1; }
    uint64_t c[2 * N_CAT];
    if (oracle_flagstat(in, c)) { fprintf(stderr, "%s\n", oracle_flagstat_error()); return 1; }
    param("in total (QC-passed reads + QC-failed reads)", c + 2 * TOTAL, tab);       /* flagstat.d:131-143 */
    param("secondary", c + 2 * SECONDARY, tab);
    param("supplementary", c + 2 * SUPPLEMENTARY, tab);
    param("duplicates", c + 2 * DUPLICATES, tab);
    param_pct("mapped", c + 2 * MAPPED, c + 2 * TOTAL, tab);
    param("paired in sequencing", c + 2 * PAIRED, tab);
    param("read1", c + 2 * READ1, tab);
    param("read2", c + 2 * READ2, tab);
    param_pct("properly paired", c + 2 * PROPER_PAIR, c + 2 * PAIRED, tab);
    param("with itself and mate mapped", c + 2 * BOTH_MAPPED, tab);
    param_pct("singletons", c + 2 * SINGLETONS, c + 2 * PAIRED, tab);
    param("with mate mapped to a different chr", c + 2 * MATE_DIFF_CHR, tab);
    param("with mate mapped to a different chr (mapQ>=5)", c + 2 * MATE_DIFF_CHR_MAPQ5, tab);
    return 0;
}
#endif
