// inflate_core.cuh -- raw DEFLATE (RFC 1951) decoder for one BGZF block, written so that ONE
// CUDA LANE decodes ONE block with its Huffman tables in (lane-interleaved) shared memory.
//
// Replaces: BioD/bio/core/bgzf/block.d:127-216 (decompressBgzfBlock -> zlib inflateInit2(-15)/
// inflate(Z_FINISH)/inflateEnd, bound through BioD/bio/core/utils/zlib.d:143-162).  The
// arithmetic being restated is zlib's (third-party, not in the sambamba sources); RFC 1951 output
// is deterministic so any correct inflater is bit-identical.
//
// Design (see DESIGN.md "K1").  A warp-per-block decoder issues ~200 instructions per symbol
// with one useful lane; giving every lane its own block makes those instructions decode 32
// symbols.  Consequences:
//  * Per-lane state bounds occupancy, and the kernel is instruction-latency bound, so tables are
//    tiny and there is NO lookup table: decoding is canonical-Huffman arithmetic.  Measured on BAM
//    data a first-level LUT misses on 5-10 % of symbols, i.e. in ~97 % of 32-lane iterations, so
//    its fast path would almost never save the warp anything while costing 4x the shared memory.
//      len = 1 + #{ j in 1..14 : peek15 >= lim[j] }      lim[] (left-justified) in REGISTERS
//      sym = sorted[ (peek15 >> (15-len)) + delta[len] ]  two shared-memory loads
//  * The SIMT loop is a flat state machine: each iteration a lane either decodes ONE symbol or
//    moves ONE 4-byte round of a pending LZ77 copy, so no lane waits for another lane's match,
//    and every iteration ends in a ballot that re-converges the warp.
//  * Output is assembled a 32-bit word at a time in a register; complete words go to a 16-word
//    per-lane ring in shared memory, complete 16-byte lines leave as one aligned 16-byte global
//    store.  Matches at distance 8..24 are served from the ring, farther ones from global memory with two
//    4-byte cp.async copies into shared memory that are consumed one iteration later, after the next symbol
//    has been decoded, so the L2/DRAM round trip overlaps the Huffman arithmetic.  The compressed input arrives
//    through a two-slot 16-byte cp.async FIFO per lane.
//    Distances below 8 (run-length style) take a byte-serial path.
//  per lane: 288 x 10-bit litlen symbols (96 w) + 15 x i16 delta (8 w) + 32 x u8 dist symbols
//            (8 w) + delta (8 w) + ring (8 w) + far landing zone (2 w) = 130 words, + 32 B input FIFO
//            = 552 B; 17.25 KB per warp; 12 warps/SM.
//
// The code is __host__ __device__ so the exact same logic is unit-tested on the CPU against zlib
// (tests/test_emul_inflate.py); the product only ever calls it from kernels.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define BD_HD __host__ __device__ __forceinline__
#define BD_HD_COLD __host__ __device__ __noinline__      // rare paths: keep them out of the hot loop's code and registers
#else
#define BD_HD inline
#define BD_HD_COLD inline
#endif

namespace bdk {

#ifdef BD_INFLATE_STATS
struct InflateStats { unsigned long long lits, matches, match_bytes, tables, near_matches, iters, len_hist[16], mlen_hist[16]; };
extern InflateStats g_inflate_stats;
#define BD_STAT(x) (x)
#else
#define BD_STAT(x) ((void)0)
#endif

enum InflateStatus : int {
    INF_OK = 0,
    INF_ERR_BTYPE = 2,       // reserved block type 3
    INF_ERR_STORED = 3,      // LEN != ~NLEN
    INF_ERR_TABLE = 4,       // over-subscribed / incomplete / missing EOB / bad repeat
    INF_ERR_CODE = 5,        // invalid code in stream
    INF_ERR_DIST = 6,        // distance too far back
    INF_ERR_OVERRUN = 7,     // output would exceed isize
    INF_ERR_SHORT = 8,       // stream ended with fewer than isize bytes
    INF_ERR_INPUT = 9        // ran past the end of the compressed data
};

// word offsets of the per-lane table regions
constexpr int T_LL_SYMS = 0;       // 288 x 10 bit, three per word
constexpr int T_LL_DELTA = 96;     // 15 x i16 (index len-1), padded to 16
constexpr int T_D_SYMS = 104;      // 32 x u8
constexpr int T_D_DELTA = 112;     // 15 x i16
constexpr int T_RING = 120;        // output ring: the last 8 complete words
constexpr int RING_WORDS = 8;
constexpr int T_FAR = T_RING + RING_WORDS;     // 2 words: landing zone of the asynchronous far-match fetch
constexpr int T_WORDS = T_FAR + 2;             // 130 lane-interleaved words
constexpr int FIFO_BYTES_PER_LANE = 32;        // two 16-byte slots of compressed input per lane (lane-major, after the interleaved words)
constexpr int SMEM_BYTES_PER_WARP = T_WORDS * 128 + 32 * FIFO_BYTES_PER_LANE;   // 17,664 B -> one 13-warp CTA per SM (kernels.cuh)
constexpr uint32_t NEAR_MAX = 4 * (RING_WORDS - 1) - 4;   // 24: farthest distance served from the ring

// ---- table storage policies -------------------------------------------------------------
// Lane-interleaved shared memory: word w of this lane lives at base[w * 32]; every lane always
// hits its own bank, so data-dependent indices never conflict.
#if defined(__CUDA_ARCH__)
// Ampere-style asynchronous copies (LDGSTS).  Their completion is tracked by cp.async groups, NOT by the register
// scoreboard, so a copy issued at the end of one loop iteration is still in flight at the top of the next; plain
// loads whose result crosses the loop back-edge are waited for at the back-edge by the compiler (that wait was
// the largest single stall reason of the one-phase decoder's loop).
__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(saddr), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_async4(uint32_t saddr, const void* g) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(saddr), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }
__device__ __forceinline__ uint32_t lds32(uint32_t saddr) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr) : "memory"); return v; }
#endif

struct SmemTab {
    uint32_t* base;
    uint32_t fifo_sa;      // shared-space address of this lane's input slot 0 (slot 1 at +512)
    uint32_t far_sa;       // shared-space address of this lane's far-fetch word 0 (word 1 at +128)
    BD_HD uint32_t ldw(int w) const { return base[w * 32]; }
    BD_HD void stw(int w, uint32_t v) const { base[w * 32] = v; }
    BD_HD uint32_t ring_ldw(uint32_t widx) const { return base[(T_RING + (widx & (RING_WORDS - 1))) * 32]; }
    BD_HD void ring_stw(uint32_t widx, uint32_t v) const { base[(T_RING + (widx & (RING_WORDS - 1))) * 32] = v; }
};
// Plain array (host tests).
struct FlatTab {
    uint32_t* base;
    uint32_t fifo_sa = 0, far_sa = 0;
    BD_HD uint32_t ldw(int w) const { return base[w]; }
    BD_HD void stw(int w, uint32_t v) const { base[w] = v; }
    BD_HD uint32_t ring_ldw(uint32_t widx) const { return base[T_RING + (widx & (RING_WORDS - 1))]; }
    BD_HD void ring_stw(uint32_t widx, uint32_t v) const { base[T_RING + (widx & (RING_WORDS - 1))] = v; }
};

template <class Tab> BD_HD uint32_t tab_ld16(const Tab& t, int region, int i) {
    uint32_t w = t.ldw(region + (i >> 1));
    return (i & 1) ? (w >> 16) : (w & 0xFFFFu);
}
template <class Tab> BD_HD void tab_st16(const Tab& t, int region, int i, uint32_t v) {
    int wi = region + (i >> 1);
    uint32_t w = t.ldw(wi);
    w = (i & 1) ? ((w & 0x0000FFFFu) | (v << 16)) : ((w & 0xFFFF0000u) | (v & 0xFFFFu));
    t.stw(wi, w);
}
template <class Tab> BD_HD uint32_t tab_ld8(const Tab& t, int region, int i) {
    return (t.ldw(region + (i >> 2)) >> ((i & 3) * 8)) & 0xFFu;
}
template <class Tab> BD_HD void tab_st8(const Tab& t, int region, int i, uint32_t v) {
    int wi = region + (i >> 2), sh = (i & 3) * 8;
    uint32_t w = t.ldw(wi);
    t.stw(wi, (w & ~(0xFFu << sh)) | ((v & 0xFFu) << sh));
}

// 10-bit entries, three per word
template <class Tab> BD_HD uint32_t tab_ld10(const Tab& t, int region, int i) {
    uint32_t q = ((uint32_t)i * 0xAAABu) >> 17;          // i / 3 for i < 2^15
    return (t.ldw(region + (int)q) >> (((uint32_t)i - 3 * q) * 10)) & 0x3FFu;
}
template <class Tab> BD_HD void tab_st10(const Tab& t, int region, int i, uint32_t v) {
    uint32_t q = ((uint32_t)i * 0xAAABu) >> 17, sh = ((uint32_t)i - 3 * q) * 10;
    uint32_t w = t.ldw(region + (int)q);
    t.stw(region + (int)q, (w & ~(0x3FFu << sh)) | ((v & 0x3FFu) << sh));
}

BD_HD uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t shift_bits) {   // low 32 bits of (hi:lo) >> shift, shift in [0,32)
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, shift_bits);
#else
    return (uint32_t)((((uint64_t)hi << 32) | lo) >> shift_bits);
#endif
}

BD_HD uint32_t bitrev32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __brev(x);
#else
    x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
    x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2);
    x = ((x >> 4) & 0x0F0F0F0Fu) | ((x & 0x0F0F0F0Fu) << 4);
    x = ((x >> 8) & 0x00FF00FFu) | ((x & 0x00FF00FFu) << 8);
    return (x >> 16) | (x << 16);
#endif
}

// ---- bit reader: 64-bit reservoir.  On the device the compressed bytes arrive through a two-slot, 16-byte
// cp.async FIFO in shared memory (every 32-byte DRAM sector is fetched once or twice instead of eight times,
// 16-32 bytes ahead of use); on the host (tests) it reads the words directly.
struct BitReader {
    uint64_t bb;
    int bc;
#if defined(__CUDA_ARCH__)
    const uint8_t* gnext;   // next 16-byte chunk to prefetch
    uint32_t fifo_sa, widx, consumed, limit_words;
    __device__ __forceinline__ uint32_t next_word() {
        if ((widx & 3) == 0) cp_async_wait<1>();       // entering a slot: its refill is older than the newest group
        uint32_t slot = fifo_sa + ((widx & 4) ? 512u : 0u);
        uint32_t w = lds32(slot + (widx & 3) * 4);
        if ((widx & 3) == 3) { cp_async16(slot, gnext); cp_async_commit(); gnext += 16; }
        widx = (widx + 1) & 7; consumed++;
        return w;
    }
    __device__ __forceinline__ void init(const uint32_t* words, uint64_t byte_off, uint32_t nbytes, uint32_t fifo_shared_addr) {
        const uint8_t* g0 = reinterpret_cast<const uint8_t*>(words) + (byte_off & ~15ull);
        fifo_sa = fifo_shared_addr;
        cp_async16(fifo_sa, g0); cp_async_commit(); cp_async16(fifo_sa + 512, g0 + 16); cp_async_commit();
        gnext = g0 + 32; cp_async_wait<0>();
        widx = (uint32_t)(byte_off & 15) >> 2; consumed = 0;
        limit_words = (uint32_t)(((byte_off & 15) + nbytes + 3) >> 2) + 3;
        unsigned mis = (unsigned)(byte_off & 3);
        bb = (uint64_t)next_word() >> (8 * mis);
        bc = 32 - 8 * (int)mis;
    }
    __device__ __forceinline__ void refill() { if (bc <= 32) { bb |= (uint64_t)next_word() << bc; bc += 32; } }   // afterwards bc >= 33
    __device__ __forceinline__ bool overrun() const { return consumed > limit_words; }
#else
    const uint32_t* wp;     // address of the prefetched word
    const uint32_t* wend;   // one past the last word that may contain stream bits
    uint32_t nw;
    void init(const uint32_t* words, uint64_t byte_off, uint32_t nbytes, uint32_t) {
        wp = words + (byte_off >> 2);
        wend = words + ((byte_off + nbytes + 3) >> 2);
        unsigned mis = (unsigned)(byte_off & 3);
        bb = (uint64_t)(*wp++) >> (8 * mis);
        bc = 32 - 8 * (int)mis;
        nw = *wp;
    }
    void refill() { if (bc <= 32) { bb |= (uint64_t)nw << bc; bc += 32; nw = *++wp; } }
    bool overrun() const { return wp > wend + 3; }
#endif
    BD_HD uint32_t lo32() const { return (uint32_t)bb; }
    BD_HD void align_byte() { drop(bc & 7); }
    BD_HD uint32_t peek(int n) const { return (uint32_t)bb & ((1u << n) - 1u); }
    BD_HD void drop(int n) { bb >>= n; bc -= n; }
    BD_HD uint32_t get(int n) { uint32_t v = peek(n); drop(n); return v; }
};

// Left-justified 15-bit limits, index len-1 (v[14] == 32768 for a complete code), built in next_block.
struct HuffLim { uint32_t v[15]; };
// The same limits packed two per register for the hot loop: pk[p] = lim[2p] | lim[2p+1] << 16, with a
// dummy 16th limit of 0x8000 (never reached: peek15 <= 0x7FFF).
struct HuffPk { uint32_t pk[8]; };

// number of j in 0..15 with rev15 >= limit j.  Guard-bit subtraction: (0x8000 | rev) - lim keeps bit 15
// set iff rev >= lim (lim <= 0x8000), two limits per 32-bit subtract; the 16 guard bits are gathered with
// sign-replicating byte permutes and counted with one POPC.  18 instructions, no dependent chain.
BD_HD int count_ge16(uint32_t rev15, const HuffPk& h) {
#if defined(__CUDA_ARCH__)
    uint32_t x = rev15 * 0x00010001u + 0x80008000u;
    uint32_t t0 = x - h.pk[0], t1 = x - h.pk[1], t2 = x - h.pk[2], t3 = x - h.pk[3];
    uint32_t t4 = x - h.pk[4], t5 = x - h.pk[5], t6 = x - h.pk[6], t7 = x - h.pk[7];
    uint32_t a, b, c, d;
    asm("prmt.b32 %0, %1, %2, 0xFDB9;" : "=r"(a) : "r"(t0), "r"(t1));   // sign-fill of bytes 1,3 of each word
    asm("prmt.b32 %0, %1, %2, 0xFDB9;" : "=r"(b) : "r"(t2), "r"(t3));
    asm("prmt.b32 %0, %1, %2, 0xFDB9;" : "=r"(c) : "r"(t4), "r"(t5));
    asm("prmt.b32 %0, %1, %2, 0xFDB9;" : "=r"(d) : "r"(t6), "r"(t7));
    uint32_t m = (a & 0x01010101u) | (b & 0x02020202u) | (c & 0x04040404u) | (d & 0x08080808u);
    return __popc(m);
#else
    int n = 0;
    for (int p = 0; p < 8; p++) { n += rev15 >= (h.pk[p] & 0xFFFFu); n += rev15 >= (h.pk[p] >> 16); }
    return n;
#endif
}

// Build one canonical table from code lengths lens[0..n).  KIND 0 = litlen (u16 symbols),
// 1 = dist (u8 symbols).  Mirrors zlib inflate_table()'s validity rules: over-subscribed ->
// error; incomplete -> error unless the longest code is <= 1 bit (dist may also be empty).
// 16 counters of 16 bits in four 64-bit registers, indexed by a run-time code length: a `uint32_t cnt[16]` indexed
// by lens[s] lives in local memory, and counting through it is a store->load dependency chain per symbol (the single
// hottest source line of K1 before this: 4.5 % of all samples for 0.7 % of the instructions).
struct Pack16x16 {
    uint64_t w[4];
    BD_HD void clear() { w[0] = w[1] = w[2] = w[3] = 0; }
    BD_HD uint32_t get(uint32_t i) const {
        uint64_t v = (i & 8) ? ((i & 4) ? w[3] : w[2]) : ((i & 4) ? w[1] : w[0]);
        return (uint32_t)(v >> ((i & 3) * 16)) & 0xFFFFu;
    }
    BD_HD void add(uint32_t i, uint32_t d) {
        uint64_t inc = (uint64_t)d << ((i & 3) * 16); uint32_t k = i >> 2;
        w[0] += k == 0 ? inc : 0; w[1] += k == 1 ? inc : 0; w[2] += k == 2 ? inc : 0; w[3] += k == 3 ? inc : 0;
    }
};

template <class Tab, int KIND>
BD_HD int build_table(const Tab& t, const uint8_t* lens, int n, HuffLim& lim) {
    Pack16x16 pc; pc.clear();
    {   // count a word (4 symbols) at a time once the pointer is 4-byte aligned (the distance lengths start mid-word)
        int s = 0;
        while (s < n && (reinterpret_cast<uintptr_t>(lens + s) & 3)) { pc.add(lens[s] & 15u, 1); s++; }
        for (; s + 4 <= n; s += 4) { uint32_t w4 = *reinterpret_cast<const uint32_t*>(lens + s); pc.add(w4 & 15u, 1); pc.add((w4 >> 8) & 15u, 1); pc.add((w4 >> 16) & 15u, 1); pc.add((w4 >> 24) & 15u, 1); }
        for (; s < n; s++) pc.add(lens[s] & 15u, 1);
    }
    uint32_t cnt[16];
#pragma unroll
    for (int i = 0; i < 16; i++) cnt[i] = pc.get((uint32_t)i);
    int left = 1, maxl = 0;
#pragma unroll
    for (int l = 1; l <= 15; l++) { left <<= 1; left -= (int)cnt[l]; if (cnt[l]) maxl = l; }
    {   // over-subscription can only be detected reliably per level; redo exactly
        int lf = 1; bool over = false;
#pragma unroll
        for (int l = 1; l <= 15; l++) { lf <<= 1; lf -= (int)cnt[l]; if (lf < 0) over = true; }
        if (over) return INF_ERR_TABLE;
    }
    if (left > 0 && (KIND == 0 ? maxl != 1 : maxl > 1)) return INF_ERR_TABLE;
    Pack16x16 nxt; nxt.clear();      // next free slot in the sorted table per length
    uint32_t code = 0, o = 0;
#pragma unroll
    for (int l = 1; l <= 15; l++) {
        nxt.add((uint32_t)l, o);
        lim.v[l - 1] = (code + cnt[l]) << (15 - l);
        int delta = (int)o - (int)code;
        tab_st16(t, KIND == 0 ? T_LL_DELTA : T_D_DELTA, l - 1, (uint32_t)delta & 0xFFFFu);
        o += cnt[l];
        code = (code + cnt[l]) << 1;
    }
    for (int s = 0; s < n; s++) {
        uint32_t l = lens[s];
        if (!l) continue;
        uint32_t slot = nxt.get(l); nxt.add(l, 1);
        if (KIND == 0) tab_st10(t, T_LL_SYMS, (int)slot, (uint32_t)s); else tab_st8(t, T_D_SYMS, (int)slot, (uint32_t)s);
    }
    return INF_OK;
}

// Decode the symbol at the bottom of `bits` (the low 32 bits of the reservoir, >= 15 of them valid) without
// consuming anything: returns the symbol (-1 on an invalid code) and its length in L.
template <class Tab, int KIND>
BD_HD int decode_sym_at(const Tab& t, const HuffPk& lim, uint32_t bits, int& L) {
    uint32_t rev15 = bitrev32(bits) >> 17;
    L = 1 + count_ge16(rev15, lim);          // code length; 16 means "beyond the last code"
    if (L > 15) return -1;
    int delta = (int)(int16_t)tab_ld16(t, KIND == 0 ? T_LL_DELTA : T_D_DELTA, L - 1);
    int idx = (int)(rev15 >> (15 - L)) + delta;
    if (idx < 0 || idx >= (KIND == 0 ? 288 : 32)) return -1;
    BD_STAT(KIND == 0 ? g_inflate_stats.len_hist[L]++ : 0);
    return KIND == 0 ? (int)tab_ld10(t, T_LL_SYMS, idx) : (int)tab_ld8(t, T_D_SYMS, idx);
}
// Decode one symbol of a canonical code.  Returns -1 on an invalid code; consumes its bits.
template <class Tab, int KIND>
BD_HD int decode_sym(const Tab& t, const HuffPk& lim, BitReader& br) {
    int L; int sym = decode_sym_at<Tab, KIND>(t, lim, (uint32_t)br.bb, L);
    if (sym >= 0) br.drop(L);
    return sym;
}

// Read the dynamic-block header and produce lens[] (RFC 1951 3.2.7).  lens must hold 320 bytes.
// The 19-symbol code-length code lives entirely in registers.
template <class BR>
BD_HD int read_dynamic_lens(BR& br, uint8_t* lens, int& nlen, int& ndist) {
    br.refill();
    nlen = (int)br.get(5) + 257;
    ndist = (int)br.get(5) + 1;
    int ncode = (int)br.get(4) + 4;
    if (nlen > 286 || ndist > 30) return INF_ERR_TABLE;
    uint64_t cl = 0;    // 19 x 3-bit lengths indexed by symbol
    const uint8_t ord[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    for (int i = 0; i < ncode; i++) { br.refill(); cl |= (uint64_t)br.get(3) << (3 * ord[i]); }
    uint32_t cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = 0; s < 19; s++) cnt[(cl >> (3 * s)) & 7]++;
    {
        int left = 1;
        for (int l = 1; l <= 7; l++) { left <<= 1; left -= (int)cnt[l]; if (left < 0) return INF_ERR_TABLE; }
        if (left > 0) return INF_ERR_TABLE;     // zlib: an incomplete code-length code is always an error
    }
    uint32_t first[8], lim[8], offs[8];
    { uint32_t code = 0, o = 0; for (int l = 1; l <= 7; l++) { first[l] = code; offs[l] = o; o += cnt[l]; lim[l] = (code + cnt[l]) << (7 - l); code = (code + cnt[l]) << 1; } }
    uint64_t dpk = 0;                         // offs[L] - first[L] as int8 per length (a first[]/offs[] pair indexed by L lives in local memory)
    for (int l = 1; l <= 7; l++) dpk |= (uint64_t)(uint8_t)(int8_t)((int)offs[l] - (int)first[l]) << (8 * l);
    uint64_t sorted_lo = 0, sorted_hi = 0;   // 19 x 5-bit symbols sorted by (len, sym)
    {
        uint32_t nx[8]; for (int l = 1; l <= 7; l++) nx[l] = offs[l];
        for (int s = 0; s < 19; s++) {
            uint32_t l = (uint32_t)(cl >> (3 * s)) & 7; if (!l) continue;
            uint32_t pos = nx[l]++;
            if (pos < 12) sorted_lo |= (uint64_t)s << (5 * pos); else sorted_hi |= (uint64_t)s << (5 * (pos - 12));
        }
    }
    int n = 0, total = nlen + ndist;
    while (n < total) {
        br.refill();
        uint32_t rev7 = bitrev32(br.lo32()) >> 25;
        int L = 1;
#pragma unroll
        for (int j = 1; j <= 6; j++) L += (rev7 >= lim[j]) ? 1 : 0;
        if (rev7 >= lim[7]) return INF_ERR_TABLE;
        uint32_t idx = (rev7 >> (7 - L)) + (uint32_t)(int32_t)(int8_t)(dpk >> (8 * L));      // - first[L] + offs[L], from a register
        if (idx >= 19) return INF_ERR_TABLE;
        uint32_t sym = (idx < 12) ? (uint32_t)(sorted_lo >> (5 * idx)) & 31u : (uint32_t)(sorted_hi >> (5 * (idx - 12))) & 31u;
        br.drop(L);
        if (sym < 16) { lens[n++] = (uint8_t)sym; continue; }
        uint32_t rep, val = 0;
        if (sym == 16) { if (n == 0) return INF_ERR_TABLE; val = lens[n - 1]; rep = 3 + br.get(2); }
        else if (sym == 17) rep = 3 + br.get(3);
        else rep = 11 + br.get(7);
        if (n + (int)rep > total) return INF_ERR_TABLE;
        while (rep--) lens[n++] = (uint8_t)val;
    }
    if (lens[256] == 0) return INF_ERR_TABLE;   // zlib: "invalid code -- missing end-of-block"
    return INF_OK;
}

// Output policy: the whole inflated stream as a byte array (global memory on the device).
// Addresses are ABSOLUTE stream offsets; put16 needs a 16-byte-aligned offset.
struct ByteOut {
    uint8_t* p;
    BD_HD void put(uint64_t i, uint32_t v) const { p[i] = (uint8_t)v; }
    BD_HD uint32_t get(uint64_t i) const { return p[i]; }
    BD_HD uint32_t getw(uint64_t widx) const { return reinterpret_cast<const uint32_t*>(p)[widx]; }   // aligned word
    BD_HD void put16(uint64_t i, uint32_t a, uint32_t b, uint32_t c, uint32_t d) const {
#if defined(__CUDA_ARCH__)
        *reinterpret_cast<uint4*>(p + i) = make_uint4(a, b, c, d);
#else
        uint32_t w[4] = {a, b, c, d};
        for (int k = 0; k < 16; k++) p[i + k] = (uint8_t)(w[k >> 2] >> ((k & 3) * 8));
#endif
    }
};

enum { ST_HDR = 0, ST_SYM = 1, ST_STORED = 2, ST_DONE = 3 };

// Warp convergence.  Lanes take different paths through an iteration (literal / match / header)
// and finish their blocks at different times.  With independent thread scheduling nothing forces
// them back together, and the first version of this kernel ran with 1.02 active threads per
// instruction.  Every iteration therefore ends in a ballot over
// the lanes still decoding: it is both the reconvergence point and the next iteration's mask.
#if defined(__CUDA_ARCH__)
#define BD_BALLOT(mask, pred) __ballot_sync((mask), (pred))
#define BD_SYNCWARP(mask) __syncwarp(mask)
#else
#define BD_BALLOT(mask, pred) ((pred) ? 1u : 0u)
#define BD_SYNCWARP(mask) ((void)0)
#endif

// Output assembly state: `cur` holds the bytes of the word being filled (absolute alignment).
struct OutState { uint32_t cur; uint32_t opos; };

// First line of a block that does not start on a 16-byte boundary: the line is shared with the
// previous block, so only this block's bytes are written, one by one.
template <class Tab, class Out>
BD_HD_COLD void flush_partial_line(Tab t, Out out, uint32_t widx, uint32_t last_word, uint64_t a0) {
    uint64_t line = ((uint64_t)(widx - 3)) << 2;
    for (uint64_t a = a0; a < line + 16; a++) {
        uint32_t w = (uint32_t)(a >> 2) == widx ? last_word : t.ring_ldw((uint32_t)(a >> 2));
        out.put(a, (w >> ((a & 3) * 8)) & 0xFFu);
    }
}

// Append n (1..4) bytes held in the low bytes of d (upper bytes zero).  a0 < 2^34 so word indices fit 32 bits.
// A completed word goes to the ring; a completed 16-byte line leaves as one aligned 16-byte store.
template <class Tab, class Out>
BD_HD void append_bytes(const Tab& t, const Out& out, OutState& os, uint64_t a0, uint32_t d, uint32_t n) {
    uint64_t A = a0 + os.opos; uint32_t k = (uint32_t)A & 3;
    uint64_t tt = (uint64_t)d << (8 * k);
    uint32_t lo = os.cur | (uint32_t)tt;
    if (k + n >= 4) {
        uint32_t widx = (uint32_t)(A >> 2);
        t.ring_stw(widx, lo);
        if ((widx & 3) == 3) {
            uint64_t line = ((uint64_t)(widx - 3)) << 2;
            if (line >= a0) out.put16(line, t.ring_ldw(widx - 3), t.ring_ldw(widx - 2), t.ring_ldw(widx - 1), lo);
            else flush_partial_line(t, out, widx, lo, a0);
        }
        os.cur = (uint32_t)(tt >> 32);
    } else os.cur = lo;
    os.opos += n;
}

// byte at absolute address A < a0 + opos (in the word being filled or in the ring)
template <class Tab>
BD_HD uint32_t recent_byte(const Tab& t, const OutState& os, uint64_t a0, uint64_t A) {
    uint32_t w = (uint32_t)(A >> 2) == (uint32_t)((a0 + os.opos) >> 2) ? os.cur : t.ring_ldw((uint32_t)(A >> 2));
    return (w >> (((uint32_t)A & 3) * 8)) & 0xFFu;
}

// Parse block headers until a block with content (or the end) is reached and build its tables.
// Cold and out of line; the 30 Huffman limits are handed back through lim16 (the lens scratch), because a
// by-reference HuffLim would force the hot loop's limit registers into local memory.
struct HdrResult { BitReader br; int rc; int state; uint32_t bfinal, stored_rem; };
// Everything is passed and returned BY VALUE: a by-reference BitReader would pin the hot loop's bit reservoir to
// local memory (its address would escape into this out-of-line call).
template <class Tab>
BD_HD_COLD HdrResult next_block(Tab t, BitReader br, uint8_t* lens, uint32_t* limpk /* 16 words */, uint32_t pos, uint32_t isize) {
    HdrResult r; r.rc = INF_OK; r.state = ST_HDR; r.bfinal = 0; r.stored_rem = 0;
    while (r.state == ST_HDR) {
        br.refill();
        r.bfinal = br.get(1); uint32_t btype = br.get(2);
        if (btype == 0) {
            br.drop(br.bc & 7);
            br.refill();
            uint32_t len = br.get(16); br.refill(); uint32_t nlen = br.get(16);
            if ((len ^ 0xFFFFu) != nlen) { r.rc = INF_ERR_STORED; break; }
            if (pos + len > isize) { r.rc = INF_ERR_OVERRUN; break; }
            r.stored_rem = len;
            r.state = len ? ST_STORED : (r.bfinal ? ST_DONE : ST_HDR);
        } else if (btype == 3) {
            r.rc = INF_ERR_BTYPE; break;
        } else {
            int nl, nd;
            if (btype == 1) {
                // fixed code (RFC 1951 3.2.6): complete over 288 litlen / 32 distance symbols; litlen 286/287
                // and distance 30/31 are rejected after decoding, as zlib does
                nl = 288; nd = 32;
                for (int i = 0; i < 144; i++) lens[i] = 8;
                for (int i = 144; i < 256; i++) lens[i] = 9;
                for (int i = 256; i < 280; i++) lens[i] = 7;
                for (int i = 280; i < 288; i++) lens[i] = 8;
                for (int i = 0; i < 32; i++) lens[288 + i] = 5;
            } else {
                int rc = read_dynamic_lens(br, lens, nl, nd);
                if (rc) { r.rc = rc; break; }
            }
            BD_STAT(g_inflate_stats.tables++);
            HuffLim ll, dd;
            int rc = build_table<Tab, 0>(t, lens, nl, ll);
            if (!rc) rc = build_table<Tab, 1>(t, lens + nl, nd, dd);
            if (rc) { r.rc = rc; break; }
            for (int p2 = 0; p2 < 8; p2++) {
                limpk[p2] = ll.v[2 * p2] | ((p2 < 7 ? ll.v[2 * p2 + 1] : 0x8000u) << 16);
                limpk[8 + p2] = dd.v[2 * p2] | ((p2 < 7 ? dd.v[2 * p2 + 1] : 0x8000u) << 16);
            }
            r.state = ST_SYM;
        }
        if (br.overrun()) { r.rc = INF_ERR_INPUT; break; }
    }
    r.br = br;
    return r;
}

// Inflate one raw-deflate stream.  words/byte_off/nbytes locate the compressed data inside a
// 4-byte-aligned buffer that has >= 64 readable bytes after the last block.  The block's isize
// output bytes go to absolute stream offsets [a0, a0+isize) of `out`.  On the device ALL 32 lanes
// of the warp must call this together; lanes without a block pass active = false.
// scratch: 320 bytes for code lengths + 64 bytes for the limit hand-over, 4-byte aligned.
// LIT3 (EXPERIMENT, kernels.cuh k1_inflate_lit3): after two literals take a third one in the same iteration when the bits
// that are left hold its whole code.  Host emulation on the bench workload: a third literal is available in 40 % of the
// iterations (about a fifth fewer iterations) for one more decode_sym_at per iteration.
template <class Tab, class Out, bool LIT3 = false>
BD_HD int inflate_block(const Tab& t, const uint32_t* words, uint64_t byte_off, uint32_t nbytes, const Out& out, uint64_t a0, uint32_t isize, uint32_t* scratch /* 384 B */, bool active = true) {
    unsigned mask = BD_BALLOT(0xFFFFFFFFu, active);
    if (!active) return INF_OK;
    uint8_t* lens = reinterpret_cast<uint8_t*>(scratch);
    uint32_t* limpk = scratch + 80;
    BitReader br; br.init(words, byte_off, nbytes, t.fifo_sa);
    HuffPk ll, dd;
#pragma unroll
    for (int i = 0; i < 8; i++) { ll.pk[i] = 0; dd.pk[i] = 0; }
    uint32_t pos = 0;                 // bytes decoded so far (some may still be in flight)
    OutState os{0u, 0u};              // bytes actually appended
    int state = ST_HDR, rc = INF_OK; uint32_t bfinal = 0, stored_rem = 0;
    uint32_t m_rem = 0, m_dist = 0, m_dst = 0;      // current match: bytes not yet fetched
    // In-flight bytes: every byte (literal or copied) is appended ONE ITERATION LATER, at the single append site
    // below.  For far matches p_w0/p_w1 are the raw loaded words; they are first touched after the next symbol
    // has been decoded, so the L2 round trip overlaps the Huffman arithmetic.
    uint32_t p_w0 = 0, p_w1 = 0, p_sh = 0, p_n = 0; bool p_far = false;
    for (;;) {
        BD_STAT(g_inflate_stats.iters++);
        int sym = -1; bool have_sym = false; uint32_t lit2 = 0, n_lit = 1;
        if (m_rem == 0) {
            if (state == ST_HDR) {
                HdrResult hr = next_block(t, br, lens, limpk, pos, isize);
                br = hr.br; rc = hr.rc; state = hr.state; bfinal = hr.bfinal; stored_rem = hr.stored_rem;
                if (rc) state = ST_DONE;
                else if (state == ST_SYM) {
#pragma unroll
                    for (int i = 0; i < 8; i++) { ll.pk[i] = limpk[i]; dd.pk[i] = limpk[8 + i]; }
                }
            }
            if (state == ST_SYM) {
                br.refill(); sym = decode_sym<Tab, 0>(t, ll, br); have_sym = true;
                if (sym < 0) { rc = INF_ERR_CODE; state = ST_DONE; have_sym = false; }
                else if (sym < 256 && pos + 2 <= isize) {
                    // Three of four symbols of BAM data are literals and most follow another literal: look at the
                    // next symbol too (>= 18 valid bits remain after a refill and one code) and take it in the same
                    // iteration if it is a literal.  Anything else stays in the reservoir for the next iteration.
                    int L2; int s2 = decode_sym_at<Tab, 0>(t, ll, (uint32_t)br.bb, L2);
                    if (s2 >= 0 && s2 < 256) {
                        br.drop(L2); lit2 = (uint32_t)s2; n_lit = 2;
                        if (LIT3 && pos + 3 <= isize) {      // the reservoir is zero above its bc valid bits: a code is whole iff its length fits
                            int L3; int s3 = decode_sym_at<Tab, 0>(t, ll, (uint32_t)br.bb, L3);
                            if (s3 >= 0 && s3 < 256 && L3 <= br.bc) { br.drop(L3); lit2 |= (uint32_t)s3 << 8; n_lit = 3; }
                        }
                    }
                }
            } else if (state == ST_STORED) {
                br.refill(); sym = (int)br.get(8); have_sym = true;
                if (--stored_rem == 0) state = bfinal ? ST_DONE : ST_HDR;
            }
        }
        // ---- A: the single append site
        if (p_n) {
#if defined(__CUDA_ARCH__)
            if (p_far) { cp_async_wait<0>(); p_w0 = lds32(t.far_sa); p_w1 = lds32(t.far_sa + 128); p_far = false; }
#endif
            uint32_t d = funnel_r(p_w0, p_w1, p_sh);
            if (p_n < 4) d &= (1u << (8 * p_n)) - 1u;
            append_bytes(t, out, os, a0, d, p_n);
            p_n = 0;
        }
        // ---- act on the decoded symbol
        if (have_sym) {
            if (sym < 256) {
                if (pos >= isize) { rc = INF_ERR_OVERRUN; state = ST_DONE; }
                else { BD_STAT(g_inflate_stats.lits += n_lit); p_w0 = (uint32_t)sym | (lit2 << 8); p_w1 = 0; p_sh = 0; p_n = n_lit; pos += n_lit; }
            } else if (sym == 256) {
                state = bfinal ? ST_DONE : ST_HDR;
            } else {
                uint32_t s = (uint32_t)sym - 257u;
                uint32_t len = 0, dist = 0; int ds = -1;
                if (s <= 28) {
                    if (s < 8) len = 3 + s;
                    else if (s == 28) len = 258;
                    else { uint32_t eb = (s >> 2) - 1; len = ((4 + (s & 3)) << eb) + 3 + br.get((int)eb); }
                    br.refill();
                    ds = decode_sym<Tab, 1>(t, dd, br);
                }
                if (ds >= 0 && ds <= 29) {
                    if (ds < 4) dist = 1 + (uint32_t)ds;
                    else { uint32_t eb = ((uint32_t)ds >> 1) - 1; dist = ((2 + ((uint32_t)ds & 1)) << eb) + 1 + br.get((int)eb); }
                }
                int e = INF_OK;
                if (s > 28 || ds < 0 || ds > 29) e = INF_ERR_CODE;
                else if (dist > pos) e = INF_ERR_DIST;
                else if (pos + len > isize) e = INF_ERR_OVERRUN;
                else if (br.overrun()) e = INF_ERR_INPUT;
                if (e) { rc = e; state = ST_DONE; }
                else {
                    BD_STAT(g_inflate_stats.matches++); BD_STAT(g_inflate_stats.match_bytes += len); BD_STAT(g_inflate_stats.mlen_hist[len >= 64 ? 15 : len / 4]++);
                    BD_STAT(g_inflate_stats.near_matches += dist <= NEAR_MAX);
                    m_dist = dist; m_dst = pos; m_rem = len; pos += len;
                }
            }
        }
        // ---- B: fetch one round (<= 4 bytes) of the current match.  Everything up to m_dst has been appended.
        if (m_rem) {
            uint32_t n = m_rem < 4 ? m_rem : 4;
            uint64_t head = a0 + m_dst;
            if (m_dist >= 8) {
                // the 4 source bytes lie entirely in complete words: two aligned words + funnel shift (done at A)
                uint64_t S = head - m_dist; uint32_t sw = (uint32_t)(S >> 2);
                if (m_dist <= NEAR_MAX) { p_w0 = t.ring_ldw(sw); p_w1 = t.ring_ldw(sw + 1); }
                else {
#if defined(__CUDA_ARCH__)
                    const uint32_t* gsrc = reinterpret_cast<const uint32_t*>(out.p) + sw;       // asynchronous: lands in shared memory, read at A
                    cp_async4(t.far_sa, gsrc); cp_async4(t.far_sa + 128, gsrc + 1); cp_async_commit(); p_far = true;
#else
                    p_w0 = out.getw(sw); p_w1 = out.getw((uint64_t)sw + 1);
#endif
                }
                p_sh = ((uint32_t)S & 3) * 8;
            } else {
                // run-length style.  H = the 8 bytes before head (hi = most recent 4), from the word being filled
                // and the two ring words before it.  The 4 output bytes are bytes (8-dist).. of H, with the
                // dist-periodic continuation when dist < 4.
                uint32_t hw = (uint32_t)(head >> 2), k8 = ((uint32_t)head & 3) * 8;
                uint32_t w1 = t.ring_ldw(hw - 1), w2 = t.ring_ldw(hw - 2);
                uint32_t hi = funnel_r(w1, os.cur, k8), lo = funnel_r(w2, w1, k8);
                uint32_t w;
                if (m_dist >= 4) w = m_dist == 4 ? hi : funnel_r(lo, hi, 8 * (8 - m_dist));
                else if (m_dist == 1) w = (hi >> 24) * 0x01010101u;
                else if (m_dist == 2) w = (hi >> 16) * 0x00010001u;
                else w = (hi >> 8) | ((hi >> 8) << 24);
                p_w0 = w; p_w1 = 0; p_sh = 0;
            }
            p_n = n; m_dst += n; m_rem -= n;
        }
        bool cont = !(state == ST_DONE && m_rem == 0 && p_n == 0);
        mask = BD_BALLOT(mask, cont);
        if (!cont) break;
    }
    if (rc) return rc;
    // flush the last, partial line (byte stores: the rest of the line belongs to the next block)
    {
        uint64_t e = a0 + os.opos, ls = e & ~15ull; if (ls < a0) ls = a0;
        for (uint64_t a = ls; a < e; a++) out.put(a, recent_byte(t, os, a0, a));
    }
    return (pos == isize && os.opos == isize) ? INF_OK : INF_ERR_SHORT;
}

}  // namespace bdk
