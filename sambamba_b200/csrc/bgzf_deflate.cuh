// bgzf_deflate.cuh -- BGZF members on the GPU, as BioD's bgzfCompress (bio/core/bgzf/compress.d) frames them: one CTA per member of at most
// BGZF_BLOCK uncompressed bytes, whose input sits in shared memory.
//   - level 0: one stored block (01 LEN NLEN data), byte for byte what zlib writes for a member of 65,280 bytes or fewer;
//   - levels -1 and 1-9 (one compressor for all of them): LZ77 over the member with a 32 KB window and hash chains, then one DEFLATE block,
//     stored, fixed or dynamic Huffman, whichever is smallest (as zlib's _tr_flush_block picks), codes limited to 15 bits (7 for the
//     code-length code).  The compressed bytes differ from zlib's; what they inflate to does not.
// The member's CRC32 is computed here too.  Output: member m at out + m * BGZF_SLOT, its length in out_len[m].
#pragma once
#include "launch.cuh"
#include <stdint.h>

namespace bdk {

constexpr uint32_t BGZF_BLOCK = 0xFF00;        // BGZF_BLOCK_SIZE: the most uncompressed bytes of one member
constexpr uint32_t BGZF_SLOT = 65536;          // BGZF_MAX_BLOCK_SIZE: the most bytes of one member
constexpr int DF_THREADS = 256;
constexpr uint32_t DF_HASH_BITS = 12, DF_NONE = 0xFFFFu;
constexpr uint32_t DF_WINDOW = 32768, DF_MAX_MATCH = 258;
constexpr uint32_t DF_CHAIN = 32;              // candidates tried per position
constexpr uint32_t DF_NICE = 128;              // a match this long ends the search
constexpr uint32_t DF_LAZY = 32;               // a match shorter than this is compared with the one at the next position
constexpr uint32_t DF_BACK = 64;               // how far back inside its chunk of DF_THREADS positions a position looks for its hash
constexpr uint32_t DF_IN_BYTES = BGZF_BLOCK + 16;

struct DfSmall {
    uint32_t hist_ll[288], hist_d[32], hist_cl[20];
    uint32_t crc_tab[256], seg[DF_THREADS], wsum[DF_THREADS / 32];
    uint32_t key[288]; uint16_t sym[288];      // the used symbols of the tree being built, by increasing frequency
    uint16_t code_ll[288], code_d[32], code_cl[20];
    uint8_t len_ll[288], len_d[32], len_cl[20];
    uint16_t rle[320]; uint32_t n_rle;         // the code-length sequence of the dynamic header: symbol | extra value << 5
    uint32_t hlit, hdist, hclen, hdr_bits, kind, dlen, crc, n;
};
constexpr size_t DF_SMEM = (sizeof(DfSmall) + 15) / 16 * 16 + DF_IN_BYTES + (size_t)BGZF_BLOCK * 2 + ((size_t)1 << DF_HASH_BITS) * 4 + DF_THREADS * 4;

__device__ __forceinline__ uint32_t df_multmodp(uint32_t a, uint32_t b) {      // a * b modulo the CRC-32 polynomial (bit-reflected)
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}
__device__ __forceinline__ uint32_t df_x8n(uint32_t n) {      // x^(8n) modulo the polynomial
    uint32_t p = 1u << 31, sq = 1u << 23;                     // x^0, x^8
    while (n) { if (n & 1) p = df_multmodp(sq, p); n >>= 1; if (n) sq = df_multmodp(sq, sq); }
    return p;
}
// crc32 of A || B from crc32(A), crc32(B) and |B| (zlib's crc32_combine)
__device__ __forceinline__ uint32_t df_crc_combine(uint32_t a, uint32_t b, uint32_t len_b, uint32_t op) { return len_b ? df_multmodp(op, a) ^ b : a; }
__device__ __forceinline__ uint32_t df_rev(uint32_t c, uint32_t n) { return __brev(c) >> (32 - n); }
__device__ __forceinline__ uint32_t df_len_code(uint32_t l) {      // l = match length - 3, 0..255: the lit/len symbol
    if (l < 8) return 257 + l;
    if (l == 255) return 285;
    const uint32_t e = 31 - __clz((int)l) - 2;
    return 265 + 4 * (e - 1) + ((l >> e) - 4);
}
__device__ __forceinline__ uint32_t df_len_extra(uint32_t sym) { return (sym < 265 || sym == 285) ? 0u : (sym - 261) / 4; }
__device__ __forceinline__ uint32_t df_dist_code(uint32_t d) {     // d = distance - 1, 0..32767
    if (d < 4) return d;
    const uint32_t e = 31 - __clz((int)d) - 1;
    return 2 * e + 2 + ((d >> e) & 1);
}
__device__ __forceinline__ uint32_t df_dist_extra(uint32_t c) { return c < 4 ? 0u : (c - 2) / 2; }
__device__ __forceinline__ void df_put(uint32_t* w, uint32_t pos, uint32_t v, uint32_t n) {      // n <= 16 bits of v at bit pos (LSB first)
    if (!n) return;
    const uint32_t i = pos >> 5, sh = pos & 31;
    atomicOr(&w[i], v << sh);
    if (sh + n > 32) atomicOr(&w[i + 1], v >> (32 - sh));
}

// Code lengths of freq[0, n) limited to maxbits, and their canonical codes (bit-reversed, as DEFLATE sends them).  The whole block calls it.
// Lengths: the in-place minimum-redundancy algorithm of Moffat and Katajainen over the used symbols sorted by frequency, then lengths over
// maxbits folded back until the Kraft sum is exact again.
__device__ void df_huffman(DfSmall& s, const uint32_t* freq, uint32_t n, uint32_t maxbits, uint8_t* len, uint16_t* code) {
    const uint32_t t = threadIdx.x;
    for (uint32_t i = t; i < n; i += DF_THREADS) {
        len[i] = 0;
        const uint32_t f = freq[i];
        if (!f) continue;
        uint32_t r = 0;
        for (uint32_t j = 0; j < n; j++) { const uint32_t g = freq[j]; r += (g && (g < f || (g == f && j < i))) ? 1u : 0u; }
        s.key[r] = f; s.sym[r] = (uint16_t)i;
    }
    __syncthreads();
    if (t == 0) {
        uint32_t m = 0; for (uint32_t i = 0; i < n; i++) m += freq[i] ? 1u : 0u;
        uint32_t* A = s.key;
        uint32_t num[33] = {0};
        if (m == 1) num[1] = 1;
        else if (m > 1) {
            A[0] += A[1]; uint32_t root = 0, leaf = 2;
            for (uint32_t next = 1; next < m - 1; next++) {
                if (leaf >= m || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = next; } else A[next] = A[leaf++];
                if (leaf >= m || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = next; } else A[next] += A[leaf++];
            }
            A[m - 2] = 0;
            for (int next = (int)m - 3; next >= 0; next--) A[next] = A[A[next]] + 1;
            int avbl = 1, used = 0, dpth = 0, root2 = (int)m - 2, next2 = (int)m - 1;
            while (avbl > 0) {
                while (root2 >= 0 && (int)A[root2] == dpth) { used++; root2--; }
                while (avbl > used) { A[next2--] = (uint32_t)dpth; avbl--; }
                avbl = 2 * used; dpth++; used = 0;
            }
            for (uint32_t i = 0; i < m; i++) num[A[i] < 32 ? A[i] : 32]++;
            for (uint32_t i = maxbits + 1; i <= 32; i++) { num[maxbits] += num[i]; num[i] = 0; }
            uint32_t total = 0;
            for (uint32_t i = maxbits; i > 0; i--) total += num[i] << (maxbits - i);
            while (total != (1u << maxbits)) {
                num[maxbits]--;
                for (uint32_t i = maxbits - 1; i > 0; i--) if (num[i]) { num[i]--; num[i + 1] += 2; break; }
                total--;
            }
        }
        uint32_t j = m;
        for (uint32_t i = 1; i <= maxbits; i++) for (uint32_t l = num[i]; l > 0; l--) len[s.sym[--j]] = (uint8_t)i;
        uint32_t bl[16] = {0}, nc[16]; for (uint32_t i = 0; i < n; i++) bl[len[i]]++;
        bl[0] = 0; uint32_t c = 0; for (uint32_t b = 1; b < 16; b++) { c = (c + bl[b - 1]) << 1; nc[b] = c; }
        for (uint32_t i = 0; i < n; i++) code[i] = len[i] ? (uint16_t)df_rev(nc[len[i]]++, len[i]) : 0;
    }
    __syncthreads();
}

// The best match at p that ends by b (length 0: none), by the hash chain through prev
__device__ __forceinline__ uint32_t df_match(const uint8_t* in, const uint16_t* prev, uint32_t p, uint32_t b, uint32_t* dist) {
    const uint32_t maxl = min(DF_MAX_MATCH, b - p);
    if (maxl < 3) return 0;
    uint32_t best = 2, bd = 0, c = prev[p];
    for (uint32_t depth = 0; c != DF_NONE && p - c <= DF_WINDOW && depth < DF_CHAIN; depth++) {
        if (in[c + best] == in[p + best]) {
            uint32_t l = 0; while (l < maxl && in[c + l] == in[p + l]) l++;
            if (l > best) { best = l; bd = p - c; if (l >= maxl || l >= DF_NICE) break; }
        }
        c = prev[c];
    }
    if (best < 3 || (best == 3 && bd > 4096)) return 0;      // (zlib drops a 3-byte match that far back: it costs more than its literals)
    *dist = bd; return best;
}

// Members [0, n_members): member m is in_len[m] bytes at stage + in_off[m].  tok: DF_THREADS * 256 words of scratch per CTA.  Grid: any size
// (each CTA takes members m = blockIdx.x, blockIdx.x + gridDim.x, ...); DF_THREADS threads and DF_SMEM bytes of dynamic shared memory.
__global__ void __launch_bounds__(DF_THREADS, 1) k_bgzf_deflate(const uint8_t* __restrict__ stage, const unsigned long long* __restrict__ in_off,
                                                                const uint32_t* __restrict__ in_len, uint32_t n_members, int level,
                                                                uint8_t* __restrict__ out, uint32_t* __restrict__ out_len, uint32_t* __restrict__ tok_all) {
    BD_DYN_SMEM(uint32_t, smem);
    DfSmall& s = *(DfSmall*)smem;
    uint8_t* in = (uint8_t*)smem + (sizeof(DfSmall) + 15) / 16 * 16;
    uint16_t* prev = (uint16_t*)(in + DF_IN_BYTES);
    uint32_t* words = (uint32_t*)prev;                        // the bit stream, once the parse no longer needs prev
    uint32_t* head = (uint32_t*)(prev + BGZF_BLOCK);          // head[h] = 1 + the latest position of hash h in the chunks before
    uint32_t* chunk_h = head + (1u << DF_HASH_BITS);
    uint32_t* tok = tok_all + (size_t)blockIdx.x * DF_THREADS * 256;
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    { uint32_t c = t; for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1; s.crc_tab[t] = c; }
    for (uint32_t m = blockIdx.x; m < n_members; m += gridDim.x) {
        const uint32_t n = in_len[m];
        const uint8_t* src = stage + in_off[m];
        for (uint32_t i = t; i < DF_IN_BYTES; i += DF_THREADS) in[i] = i < n ? src[i] : 0;
        for (uint32_t i = t; i < (1u << DF_HASH_BITS); i += DF_THREADS) head[i] = 0;
        for (uint32_t i = t; i < 288; i += DF_THREADS) s.hist_ll[i] = 0;
        if (t < 32) s.hist_d[t] = 0;
        if (t < 20) s.hist_cl[t] = 0;
        __syncthreads();
        // ---- CRC32: a segment of S bytes per thread, combined by warp 0
        const uint32_t S = (n + DF_THREADS - 1) / DF_THREADS;
        const uint32_t a = min(n, t * S), b = min(n, a + S);
        { uint32_t c = 0xFFFFFFFFu; for (uint32_t i = a; i < b; i++) c = s.crc_tab[(c ^ in[i]) & 0xFFu] ^ (c >> 8); s.seg[t] = ~c; }
        __syncthreads();
        if (warp == 0) {
            const uint32_t opS = df_x8n(S);
            uint32_t acc = 0, run = 0;
            for (uint32_t k = 0; k < DF_THREADS / 32; k++) {
                const uint32_t j = lane * (DF_THREADS / 32) + k, l = min(n, j * S + S) - min(n, j * S);
                acc = df_crc_combine(acc, s.seg[j], l, l == S ? opS : df_x8n(l)); run += l;
            }
            const uint32_t op8 = df_x8n(S * (DF_THREADS / 32));
            const uint32_t mine = acc;
            for (uint32_t k = 0; k < 32; k++) {
                const uint32_t c = __shfl_sync(0xFFFFFFFFu, mine, k), l = __shfl_sync(0xFFFFFFFFu, run, k);
                if (k == 0) acc = c; else acc = df_crc_combine(acc, c, l, l == S * (DF_THREADS / 32) ? op8 : df_x8n(l));
            }
            if (lane == 0) s.crc = acc;
        }
        uint32_t kind = 0;                                    // 0 stored, 1 fixed, 2 dynamic
        if (level != 0 && n) {
            // ---- hash chains: prev[p] = the latest earlier position of p's hash (within DF_BACK inside its chunk, else from the chunks before)
            for (uint32_t c0 = 0; c0 < n; c0 += DF_THREADS) {
                const uint32_t p = c0 + t;
                const uint32_t h = p + 2 < n ? ((in[p] | (uint32_t)in[p + 1] << 8 | (uint32_t)in[p + 2] << 16) * 0x9E3779B1u) >> (32 - DF_HASH_BITS) : 0xFFFFFFFFu;
                chunk_h[t] = h;
                __syncthreads();
                if (p < n) {
                    uint32_t pv = DF_NONE;
                    if (h != 0xFFFFFFFFu) {
                        for (uint32_t k = 1; k <= min(t, DF_BACK); k++) if (chunk_h[t - k] == h) { pv = p - k; break; }
                        if (pv == DF_NONE && head[h]) pv = head[h] - 1;
                    }
                    prev[p] = (uint16_t)pv;
                }
                __syncthreads();
                if (h != 0xFFFFFFFFu) atomicMax(&head[h], p + 1);
            }
            __syncthreads();
            // ---- greedy parse with one step of lazy matching, a segment per thread (matches end inside the segment)
            uint32_t* mt = tok + t * 256, nt = 0;
            {
                uint32_t p = a, d = 0, l = a < b ? df_match(in, prev, a, b, &d) : 0;
                while (p < b) {
                    if (l && l < DF_LAZY && p + 1 < b) {
                        uint32_t d2 = 0; const uint32_t l2 = df_match(in, prev, p + 1, b, &d2);
                        if (l2 > l) { mt[nt++] = in[p]; atomicAdd(&s.hist_ll[in[p]], 1u); p++; l = l2; d = d2; continue; }
                    }
                    if (l) {
                        mt[nt++] = 0x80000000u | (l - 3) << 16 | (d - 1);
                        atomicAdd(&s.hist_ll[df_len_code(l - 3)], 1u); atomicAdd(&s.hist_d[df_dist_code(d - 1)], 1u);
                        p += l;
                    } else { mt[nt++] = in[p]; atomicAdd(&s.hist_ll[in[p]], 1u); p++; }
                    l = p < b ? df_match(in, prev, p, b, &d) : 0;
                }
            }
            if (t == 0) s.hist_ll[256] = 1;
            __syncthreads();
            if (t == 0) {      // every tree gets two used symbols at least, so that each is complete (they cost nothing when unused)
                uint32_t u = 0; for (int i = 0; i < 30; i++) u += s.hist_d[i] ? 1u : 0u;
                if (u < 2) { if (!s.hist_d[0]) s.hist_d[0] = 1; else s.hist_d[1] = 1; }
                if (u == 0) s.hist_d[1] = 1;
            }
            __syncthreads();
            // ---- costs of the three block kinds; trees (dynamic: lit/len, distance, then the code-length code)
            df_huffman(s, s.hist_ll, 286, 15, s.len_ll, s.code_ll);
            df_huffman(s, s.hist_d, 30, 15, s.len_d, s.code_d);
            if (t == 0) {
                uint32_t hl = 286; while (hl > 257 && !s.len_ll[hl - 1]) hl--;
                uint32_t hd = 30; while (hd > 1 && !s.len_d[hd - 1]) hd--;
                s.hlit = hl; s.hdist = hd;
                uint8_t all[316]; for (uint32_t i = 0; i < hl; i++) all[i] = s.len_ll[i]; for (uint32_t i = 0; i < hd; i++) all[hl + i] = s.len_d[i];
                const uint32_t na = hl + hd; uint32_t nr = 0;
                for (uint32_t i = 0; i < na;) {
                    const uint8_t v = all[i]; uint32_t r = 1; while (i + r < na && all[i + r] == v) r++;
                    if (v == 0 && r >= 3) { const uint32_t k = min(r, 138u); s.rle[nr++] = k >= 11 ? (uint16_t)(18 | (k - 11) << 5) : (uint16_t)(17 | (k - 3) << 5); i += k; }
                    else if (v != 0 && r >= 4) { s.rle[nr++] = v; const uint32_t k = min(r - 1, 6u); s.rle[nr++] = (uint16_t)(16 | (k - 3) << 5); i += 1 + k; }
                    else { s.rle[nr++] = v; i++; }
                }
                s.n_rle = nr;
                for (uint32_t i = 0; i < nr; i++) s.hist_cl[s.rle[i] & 31]++;
                uint32_t u = 0; for (int i = 0; i < 19; i++) u += s.hist_cl[i] ? 1u : 0u;
                if (u < 2) s.hist_cl[s.hist_cl[0] ? 1 : 0] = 1;      // (the code-length code must be complete)
            }
            __syncthreads();
            df_huffman(s, s.hist_cl, 19, 7, s.len_cl, s.code_cl);
            if (t == 0) {
                const uint8_t ord[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
                uint32_t hc = 19; while (hc > 4 && !s.len_cl[ord[hc - 1]]) hc--;
                s.hclen = hc;
                unsigned long long dyn = 3 + 5 + 5 + 4 + 3 * hc, fix = 3, ext = 0;
                for (uint32_t i = 0; i < s.n_rle; i++) { const uint32_t v = s.rle[i] & 31; dyn += s.len_cl[v] + (v == 16 ? 2 : v == 17 ? 3 : v == 18 ? 7 : 0); }
                s.hdr_bits = (uint32_t)dyn;
                for (uint32_t i = 0; i < 286; i++) {
                    const unsigned long long f = s.hist_ll[i];
                    dyn += f * s.len_ll[i]; fix += f * (i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8); ext += f * df_len_extra(i);
                }
                for (uint32_t i = 0; i < 30; i++) { dyn += (unsigned long long)s.hist_d[i] * s.len_d[i]; fix += (unsigned long long)s.hist_d[i] * 5; ext += (unsigned long long)s.hist_d[i] * df_dist_extra(i); }
                // (the two padding distance symbols were counted once each: a few bits too many, the same for both Huffman kinds)
                const unsigned long long opt_b = (dyn + ext + 7) >> 3, fix_b = (fix + ext + 7) >> 3;
                const unsigned long long best = fix_b <= opt_b ? fix_b : opt_b;
                s.kind = (uint64_t)n + 4 <= best ? 0u : fix_b <= opt_b ? 1u : 2u;
                if (s.kind == 1) {      // the fixed codes (RFC 1951 3.2.6)
                    for (uint32_t i = 0; i < 288; i++) { const uint32_t l = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8, c = i < 144 ? 0x30 + i : i < 256 ? 0x190 + (i - 144) : i < 280 ? i - 256 : 0xC0 + (i - 280); s.len_ll[i] = (uint8_t)l; s.code_ll[i] = (uint16_t)df_rev(c, l); }
                    for (uint32_t i = 0; i < 30; i++) { s.len_d[i] = 5; s.code_d[i] = (uint16_t)df_rev(i, 5); }
                    s.hdr_bits = 3;
                }
            }
            __syncthreads();
            kind = s.kind;
            if (kind) {
                // ---- bit packing: each thread's bits from a block-wide prefix sum, OR-ed into shared words
                uint32_t mine = 0;
                for (uint32_t k = 0; k < nt; k++) {
                    const uint32_t v = mt[k];
                    if (v & 0x80000000u) { const uint32_t lc = df_len_code((v >> 16) & 0xFFu), dc = df_dist_code(v & 0xFFFFu); mine += s.len_ll[lc] + df_len_extra(lc) + s.len_d[dc] + df_dist_extra(dc); }
                    else mine += s.len_ll[v];
                }
                uint32_t incl = mine; for (uint32_t sh = 1; sh < 32; sh <<= 1) { const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, incl, sh); if (lane >= sh) incl += o; }
                if (lane == 31) s.wsum[warp] = incl;
                for (uint32_t i = t; i < BGZF_SLOT / 4 + 2; i += DF_THREADS) words[i] = 0;
                __syncthreads();
                uint32_t pos = s.hdr_bits; for (uint32_t w = 0; w < warp; w++) pos += s.wsum[w];
                pos += incl - mine;
                uint32_t body = 0; for (uint32_t w = 0; w < DF_THREADS / 32; w++) body += s.wsum[w];
                for (uint32_t k = 0; k < nt; k++) {
                    const uint32_t v = mt[k];
                    if (v & 0x80000000u) {
                        const uint32_t l = (v >> 16) & 0xFFu, d = v & 0xFFFFu, lc = df_len_code(l), dc = df_dist_code(d), le = df_len_extra(lc), de = df_dist_extra(dc);
                        df_put(words, pos, s.code_ll[lc], s.len_ll[lc]); pos += s.len_ll[lc];
                        df_put(words, pos, l & ((1u << le) - 1), le); pos += le;
                        df_put(words, pos, s.code_d[dc], s.len_d[dc]); pos += s.len_d[dc];
                        df_put(words, pos, de ? (d & ((1u << de) - 1)) : 0, de); pos += de;
                    } else { df_put(words, pos, s.code_ll[v], s.len_ll[v]); pos += s.len_ll[v]; }
                }
                if (t == 0) {
                    df_put(words, 0, 1u | kind << 1, 3);
                    uint32_t q = 3;
                    if (kind == 2) {
                        const uint8_t ord[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
                        df_put(words, q, s.hlit - 257, 5); q += 5; df_put(words, q, s.hdist - 1, 5); q += 5; df_put(words, q, s.hclen - 4, 4); q += 4;
                        for (uint32_t i = 0; i < s.hclen; i++) { df_put(words, q, s.len_cl[ord[i]], 3); q += 3; }
                        for (uint32_t i = 0; i < s.n_rle; i++) {
                            const uint32_t v = s.rle[i] & 31, x = s.rle[i] >> 5, xb = v == 16 ? 2 : v == 17 ? 3 : v == 18 ? 7 : 0;
                            df_put(words, q, s.code_cl[v], s.len_cl[v]); q += s.len_cl[v];
                            df_put(words, q, x, xb); q += xb;
                        }
                    }
                    const uint32_t e = s.hdr_bits + body;
                    df_put(words, e, s.code_ll[256], s.len_ll[256]);
                    s.dlen = (e + s.len_ll[256] + 7) >> 3;
                }
                __syncthreads();
            }
        }
        if (t == 0) s.kind = kind;
        __syncthreads();
        // ---- the member: header, DEFLATE data, CRC32, ISIZE
        uint8_t* o = out + (size_t)m * BGZF_SLOT;
        uint32_t dlen;
        if (s.kind == 0) {
            dlen = n + 5;
            for (uint32_t i = t; i < n; i += DF_THREADS) o[18 + 5 + i] = in[i];
            if (t == 0) { o[18] = 1; o[19] = (uint8_t)n; o[20] = (uint8_t)(n >> 8); o[21] = (uint8_t)~n; o[22] = (uint8_t)(~n >> 8); }
        } else {
            dlen = s.dlen;
            for (uint32_t i = t; i < dlen; i += DF_THREADS) o[18 + i] = (uint8_t)(words[i >> 2] >> (8 * (i & 3)));
        }
        if (t == 0) {
            const uint8_t hs[16] = {31, 139, 8, 4, 0, 0, 0, 0, 0, 255, 6, 0, 66, 67, 2, 0};
            for (int i = 0; i < 16; i++) o[i] = hs[i];
            const uint32_t total = 18 + dlen + 8;
            o[16] = (uint8_t)(total - 1); o[17] = (uint8_t)((total - 1) >> 8);
            uint8_t* f = o + 18 + dlen;
            for (int i = 0; i < 4; i++) { f[i] = (uint8_t)(s.crc >> (8 * i)); f[4 + i] = (uint8_t)(n >> (8 * i)); }
            out_len[m] = total;
        }
        __syncthreads();
    }
}

// Members [m0, m1) of out (BGZF_SLOT apart) packed back to back into dst, member m at coff[m] - coff[m0]; a CTA per member
__global__ void __launch_bounds__(256) k_bgzf_pack(const uint8_t* __restrict__ out, const uint32_t* __restrict__ out_len, const unsigned long long* __restrict__ coff,
                                                   uint32_t m0, uint32_t m1, uint8_t* __restrict__ dst) {
    for (uint32_t m = m0 + blockIdx.x; m < m1; m += gridDim.x) {
        const uint8_t* s = out + (size_t)m * BGZF_SLOT; uint8_t* d = dst + (coff[m] - coff[m0]);
        for (uint32_t i = threadIdx.x; i < out_len[m]; i += blockDim.x) d[i] = s[i];
    }
}

}  // namespace bdk
