// inflate2_core.cuh -- K1 in two phases (round 2).  Replaces decompressBgzfBlock (BioD/bio/core/bgzf/block.d:127-216 ->
// zlib inflate, bound in BioD/bio/core/utils/zlib.d:143-162); RFC 1951 output is deterministic, so the result is
// bit-identical to zlib's whatever the decomposition.
//
// Why two phases: the one-phase lane-per-block decoder
// (inflate_core.cuh, kept as the exact fallback and for the header blocks) executes the union of "decode a symbol",
// "append bytes", "fetch a round of an LZ77 copy" for 32 lanes in different states -- 535 instructions per iteration at
// 15 of 32 active lanes -- and every far LZ77 source is a DRAM sector of one of 57 k concurrent 32 KB windows
// (46.8 GB read for 6 GB of algorithmic bytes).  Everything that does not need the bit stream moves out of that loop:
//
//   phase 1  huff_phase   ONE LANE PER BGZF BLOCK, Huffman decoding only.  It writes two append-only streams and never
//            looks at the output: the literals, as *literal ranks*, packed back to back (16-byte stores), and one 4-byte
//            token per match {literals since the previous token, length, distance}.  No output position, no line
//            assembly, no window.  No symbol table in shared memory either: in a canonical code the symbols of one
//            length are in ascending order, literals first, so "is it a literal" is one compare of the code value against
//            a per-length threshold and the literal's rank among all literals (0..255) is one add; the rank -> byte table
//            (256 bytes per deflate block) goes to global memory and phase 2 applies it.  There is no bit reservoir: an
//            iteration takes the 64 bits at the reader's position out of a shared-memory ring (BitWin), decodes three litlen
//            codes speculatively without a branch between them, takes up to three literals, or a literal and a match, or a
//            match -- every code a funnel shift of the same two registers -- and advances the position once.  Per-lane
//            shared memory: 288 (+64) bytes instead of 552.
//            Deflate-block headers are parsed in ROUNDS: a lane that reaches an end-of-block parks until every running
//            lane of the warp has (or HDR_WAIT iterations passed), so the table building runs with many active lanes
//            instead of one (19 % of all samples sat there at 1.6 active lanes).
//   phase 2  k1_lz (kernels.cuh)   ONE WARP PER BGZF BLOCK, 32 tokens at a time: a warp scan gives every token its place in
//            the output; the group's literals are scattered there through the block's rank -> byte table (lanes stride over
//            the packed literals: coalesced reads); then the matches, lane = token, sources resolved by pointer jumping
//            through the group's own tokens, so a group's copies only read finished bytes and need no order among
//            themselves.  The warp works inside its own 64 KB of output, which its SM's L1/L2 hold: no DRAM re-reads.
//            Distances and lengths are validated here (phase 1 does not know positions).
//
// Blocks phase 1 cannot express (more than MAX_SEG deflate blocks in one BGZF block, more tokens than the token area
// holds) get status INF_FALLBACK and are decoded by the one-phase kernel (k1_fallback): exact, just slower.
#pragma once
#include "inflate_core.cuh"

namespace bdk {

constexpr int INF_FALLBACK = 100;        // phase 1 gave up on this block: the one-phase decoder takes it
constexpr int MAX_SEG = 8;               // deflate blocks per BGZF block phase 2 keeps tables for (zlib: one per 16383 symbols, 3-4 per block)
constexpr uint32_t SEG_RAW = 1u << 31;   // seg_info: the literals of this segment are bytes already (stored block, fixed code: rank == byte)
constexpr uint32_t TOK_NOMATCH = 1u << 31;   // token: `lit` literals and no match (a literal run reached LIT_RUN_MAX)
constexpr uint32_t LIT_RUN_MAX = 252;    // a run is cut by a TOK_NOMATCH token once it reaches this (<= 255 - 3: three literals per iteration)

// per-lane table words (lane-interleaved like inflate_core.cuh: word w of a lane at base[w * 32])
constexpr int H_LL = 0;          // 16 x 2 words per code length L: {thr | dl << 16, dn}:  code value t (L bits) is a literal iff t < thr,
                                 //   then its rank among the literals is (t + dl) & 0xFF; otherwise H_NL[(t + dn) & 0xFFFF] = symbol - 256
constexpr int H_NL = 32;         // 32 x u8: the non-literal symbols (256 = end of block, 257.. = lengths) by rank, minus 256
constexpr int H_DD = 40;         // 15 x i16 distance deltas (index = rank in the sorted distance symbols)
constexpr int H_DS = 48;         // 32 x u8 sorted distance symbols
constexpr int H_WORDS = 56;
constexpr int H_SMEM_BYTES_PER_WARP = H_WORDS * 128 + 32 * 64;      // tables + the input ring (BitWin): 9,216 B

// Table storage of phase 1.  LIMS (template flag of huff_phase): the 2 x 8 packed Huffman limit words live in the table
// storage too (one 16-byte quad per lane and load, [quad][lane] so that a warp's LDS.128 is conflict-free) and are loaded
// where a code is decoded, instead of occupying 16 registers for the whole kernel: their addresses do not depend on the
// bit stream, so the loads issue ahead of the decode.
struct SmemTab2 {
    uint32_t* base;        // this lane's word 0 (word w at base[w * 32])
    uint32_t* lim;         // this lane's limit quad 0 (quad q of table `which` at lim[(which * 2 + q) * 128 .. +4))
    uint32_t fifo_sa;      // shared-space address of this lane's input ring (BitWin)
    BD_HD uint32_t ldw(int w) const { return base[w * 32]; }
    BD_HD void stw(int w, uint32_t v) const { base[w * 32] = v; }
    BD_HD void st_lim(int which, const uint32_t* pk) const { for (int i = 0; i < 8; i++) lim[(which * 2 + (i >> 2)) * 128 + (i & 3)] = pk[i]; }
    BD_HD void ld_lim(int which, HuffPk& h) const {
#if defined(__CUDA_ARCH__)
        uint4 a = *reinterpret_cast<const uint4*>(lim + (which * 2) * 128), b = *reinterpret_cast<const uint4*>(lim + (which * 2 + 1) * 128);
        h.pk[0] = a.x; h.pk[1] = a.y; h.pk[2] = a.z; h.pk[3] = a.w; h.pk[4] = b.x; h.pk[5] = b.y; h.pk[6] = b.z; h.pk[7] = b.w;
#else
        for (int i = 0; i < 8; i++) h.pk[i] = lim[(which * 2 + (i >> 2)) * 128 + (i & 3)];
#endif
    }
};
struct FlatTab2 {          // plain arrays (host tests)
    uint32_t* base; uint32_t* lim; uint32_t fifo_sa = 0;
    BD_HD uint32_t ldw(int w) const { return base[w]; }
    BD_HD void stw(int w, uint32_t v) const { base[w] = v; }
    BD_HD void st_lim(int which, const uint32_t* pk) const { for (int i = 0; i < 8; i++) lim[which * 8 + i] = pk[i]; }
    BD_HD void ld_lim(int which, HuffPk& h) const { for (int i = 0; i < 8; i++) h.pk[i] = lim[which * 8 + i]; }
};
constexpr int H_LIM_BYTES_PER_WARP = 4 * 512;      // LIMS: 2 tables x 2 quads x 32 lanes x 16 B

// ---- bit window: no reservoir registers.  The compressed bytes of a lane stream through a 64-byte ring in shared memory (four
// 16-byte cp.async slots, [slot][lane]); the reader is a bit position P.  window() hands out the 64 bits at P (three ring
// words, two funnel shifts), which is more than one iteration of phase 1 consumes (three literal codes 45, or literal + length
// + extra + distance + extra 15+15+5+15+13 = 63), so every code of an iteration is a funnel shift of those two registers by a
// bit offset -- nothing is shifted out between codes -- and advance() moves P once.  When P leaves a slot, the slot is
// refilled with the bytes 64 ahead; cp.async.wait_group 2 before a window leaves at most the two slots beyond the window in
// flight.  The header code (cold) uses the same object through get / drop / lo32.  Host (tests): plain words.
constexpr int RING_SLOTS = 4;
constexpr int RING_BYTES_PER_LANE = RING_SLOTS * 16;
struct BitWin {
    uint32_t P;            // bit position, relative to the 16-byte aligned address g0
    uint32_t pend;         // first bit past the stream
#if defined(__CUDA_ARCH__)
    const uint8_t* g0; uint32_t ring_sa;      // shared-space address of this lane's slot 0 (slot k at + k * 512)
    __device__ __forceinline__ void init(const uint32_t* words, uint64_t byte_off, uint32_t nbytes, uint32_t ring_shared_addr) {
        g0 = reinterpret_cast<const uint8_t*>(words) + (byte_off & ~15ull); ring_sa = ring_shared_addr;
#pragma unroll
        for (int k = 0; k < RING_SLOTS; k++) { cp_async16(ring_sa + k * 512, g0 + 16 * k); cp_async_commit(); }
        P = 8u * (uint32_t)(byte_off & 15); pend = P + 8u * nbytes;
    }
    __device__ __forceinline__ uint32_t ring_word(uint32_t w) const { return lds32(ring_sa + ((w >> 2) & (RING_SLOTS - 1)) * 512 + (w & 3) * 4); }
    __device__ __forceinline__ void window(uint32_t& b0, uint32_t& b1) const {
        cp_async_wait<2>();
        const uint32_t wi = P >> 5, sh = P & 31;
        const uint32_t w0 = ring_word(wi), w1 = ring_word(wi + 1), w2 = ring_word(wi + 2);
        b0 = __funnelshift_r(w0, w1, sh); b1 = __funnelshift_r(w1, w2, sh);
    }
    __device__ __forceinline__ void advance(uint32_t n) {
        const uint32_t s0 = P >> 7; P += n;
        if ((P >> 7) != s0) { cp_async16(ring_sa + (s0 & (RING_SLOTS - 1)) * 512, g0 + 16 * (s0 + RING_SLOTS)); cp_async_commit(); }      // n < 128: one slot at most
    }
#else
    const uint32_t* w;     // word 0 of the aligned address
    void init(const uint32_t* words, uint64_t byte_off, uint32_t nbytes, uint32_t) { w = words + ((byte_off & ~15ull) >> 2); P = 8u * (uint32_t)(byte_off & 15); pend = P + 8u * nbytes; }
    void window(uint32_t& b0, uint32_t& b1) const {
        const uint32_t wi = P >> 5, sh = P & 31; const uint32_t w0 = w[wi], w1 = w[wi + 1], w2 = w[wi + 2];
        b0 = funnel_r(w0, w1, sh); b1 = funnel_r(w1, w2, sh);
    }
    void advance(uint32_t n) { P += n; }
#endif
    BD_HD bool overrun() const { return P > pend; }
    // the interface the header code uses (read_dynamic_lens is shared with the one-phase decoder's BitReader)
    BD_HD void refill() {}
    BD_HD uint32_t lo32() const { uint32_t b0, b1; window(b0, b1); return b0; }
    BD_HD uint32_t peek(int n) const { return lo32() & ((1u << n) - 1u); }      // n < 32
    BD_HD void drop(int n) { advance((uint32_t)n); }
    BD_HD uint32_t get(int n) { uint32_t v = peek(n); advance((uint32_t)n); return v; }
    BD_HD void align_byte() { advance((8u - (P & 7u)) & 7u); }
};
// the 32 bits at offset o (< 64) of the 64-bit window (b1:b0); at least 64 - o of them are stream bits
BD_HD uint32_t win_at(uint32_t b0, uint32_t b1, uint32_t o) { return o < 32u ? funnel_r(b0, b1, o) : (b1 >> (o & 31u)); }

// Where phase 1 leaves what phase 2 needs.
struct HuffOut {
    uint32_t* tok; uint32_t tok_cap;     // this block's token area
    uint8_t* lits;                       // this block's literal area: isize bytes, 16-byte aligned, padded to a multiple of 16
    uint8_t* lit_tab;                    // MAX_SEG x 256 bytes: literal rank -> byte, per deflate block with a dynamic code
    uint32_t* seg_info;                  // MAX_SEG words: index of the deflate block's first literal in `lits` | SEG_RAW
};

// Litlen tables of one deflate block.  Validity rules as zlib inflate_table() (and build_table in inflate_core.cuh).
template <class Tab>
BD_HD int build_litlen2(const Tab& t, const uint8_t* lens, int n, HuffLim& lim, uint8_t* lit_dst) {
    Pack16x16 pc, pl; pc.clear(); pl.clear();      // symbols per length: all, literals only
    const int nl = n < 256 ? n : 256;
    {
        int s = 0;       // lens is 4-byte aligned (the scratch array)
        for (; s + 4 <= nl; s += 4) { uint32_t w4 = *reinterpret_cast<const uint32_t*>(lens + s); pl.add(w4 & 15u, 1); pl.add((w4 >> 8) & 15u, 1); pl.add((w4 >> 16) & 15u, 1); pl.add((w4 >> 24) & 15u, 1); }
        for (; s < nl; s++) pl.add(lens[s] & 15u, 1);
        pc = pl;
        for (s = nl; s < n; s++) pc.add(lens[s] & 15u, 1);
    }
    uint32_t cnt[16], cl[16];
#pragma unroll
    for (int i = 0; i < 16; i++) { cnt[i] = pc.get((uint32_t)i); cl[i] = pl.get((uint32_t)i); }
    int left = 1, maxl = 0; bool over = false;
#pragma unroll
    for (int l = 1; l <= 15; l++) { left <<= 1; left -= (int)cnt[l]; if (left < 0) over = true; if (cnt[l]) maxl = l; }
    if (over) return INF_ERR_TABLE;
    if (left > 0 && maxl != 1) return INF_ERR_TABLE;
    Pack16x16 nx_lit, nx_nl; nx_lit.clear(); nx_nl.clear();
    uint32_t code = 0, litbase = 0, nlbase = 0;
#pragma unroll
    for (int l = 1; l <= 15; l++) {
        nx_lit.add((uint32_t)l, litbase); nx_nl.add((uint32_t)l, nlbase);
        lim.v[l - 1] = (code + cnt[l]) << (15 - l);
        uint32_t thr = code + cl[l];
        uint32_t dl = (litbase - code) & 0xFFFFu, dn = (nlbase - cl[l] - code) & 0xFFFFu;
        t.stw(H_LL + 2 * (l - 1), (thr & 0xFFFFu) | (dl << 16));
        t.stw(H_LL + 2 * (l - 1) + 1, dn);
        litbase += cl[l]; nlbase += cnt[l] - cl[l];
        code = (code + cnt[l]) << 1;
    }
    for (int s = 0; s < n; s++) {
        uint32_t l = lens[s];
        if (!l) continue;
        if (s < 256) { uint32_t slot = nx_lit.get(l); nx_lit.add(l, 1); if (lit_dst) lit_dst[slot] = (uint8_t)s; }
        else { uint32_t slot = nx_nl.get(l); nx_nl.add(l, 1); tab_st8(t, H_NL, (int)slot, (uint32_t)(s - 256)); }
    }
    return INF_OK;
}

template <class Tab>
BD_HD int build_dist2(const Tab& t, const uint8_t* lens, int n, HuffLim& lim) {
    Pack16x16 pc; pc.clear();
    for (int s = 0; s < n; s++) pc.add(lens[s] & 15u, 1);
    uint32_t cnt[16];
#pragma unroll
    for (int i = 0; i < 16; i++) cnt[i] = pc.get((uint32_t)i);
    int left = 1, maxl = 0; bool over = false;
#pragma unroll
    for (int l = 1; l <= 15; l++) { left <<= 1; left -= (int)cnt[l]; if (left < 0) over = true; if (cnt[l]) maxl = l; }
    if (over) return INF_ERR_TABLE;
    if (left > 0 && maxl > 1) return INF_ERR_TABLE;
    Pack16x16 nxt; nxt.clear();
    uint32_t code = 0, o = 0;
#pragma unroll
    for (int l = 1; l <= 15; l++) {
        nxt.add((uint32_t)l, o);
        lim.v[l - 1] = (code + cnt[l]) << (15 - l);
        tab_st16(t, H_DD, l - 1, (uint32_t)((int)o - (int)code) & 0xFFFFu);
        o += cnt[l];
        code = (code + cnt[l]) << 1;
    }
    for (int s = 0; s < n; s++) {
        uint32_t l = lens[s];
        if (!l) continue;
        uint32_t slot = nxt.get(l); nxt.add(l, 1);
        tab_st8(t, H_DS, (int)slot, (uint32_t)s);
    }
    return INF_OK;
}

// Parse block headers until a block with content (or the end) is reached; build its tables.  Cold, out of line, everything by
// value (see next_block in inflate_core.cuh).  raw: the block's literals need no translation.
struct HdrResult2 { BitWin br; int rc; int state; uint32_t bfinal, stored_rem, raw; };
template <class Tab>
BD_HD_COLD HdrResult2 next_block2(Tab t, BitWin br, uint8_t* lens, uint32_t* limpk /* 16 words */, uint8_t* lit_dst) {
    HdrResult2 r; r.rc = INF_OK; r.state = ST_HDR; r.bfinal = 0; r.stored_rem = 0; r.raw = 1;
    while (r.state == ST_HDR) {
        br.refill();
        r.bfinal = br.get(1); uint32_t btype = br.get(2);
        if (btype == 0) {
            br.align_byte();
            uint32_t len = br.get(16), nlen = br.get(16);
            if ((len ^ 0xFFFFu) != nlen) { r.rc = INF_ERR_STORED; break; }
            r.stored_rem = len; r.raw = 1;
            r.state = len ? ST_STORED : (r.bfinal ? ST_DONE : ST_HDR);
        } else if (btype == 3) {
            r.rc = INF_ERR_BTYPE; break;
        } else {
            int nl, nd;
            if (btype == 1) {
                // fixed code (RFC 1951 3.2.6).  Its literals sorted by (length, symbol) are 0..143 (8 bits) then 144..255 (9 bits):
                // rank == byte, no table needed
                nl = 288; nd = 32; r.raw = 1;
                for (int i = 0; i < 144; i++) lens[i] = 8;
                for (int i = 144; i < 256; i++) lens[i] = 9;
                for (int i = 256; i < 280; i++) lens[i] = 7;
                for (int i = 280; i < 288; i++) lens[i] = 8;
                for (int i = 0; i < 32; i++) lens[288 + i] = 5;
            } else {
                int rc = read_dynamic_lens(br, lens, nl, nd);
                if (rc) { r.rc = rc; break; }
                r.raw = 0;
            }
            HuffLim ll, dd;
            int rc = build_litlen2<Tab>(t, lens, nl, ll, r.raw ? nullptr : lit_dst);
            if (!rc) rc = build_dist2<Tab>(t, lens + nl, nd, dd);
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

// One litlen code at the bottom of `bits`: its length L (16: no such code), its code value tc and the first table word of L.
#define BD_LITLEN_PEEK(bits, L, tc, e0)                                         \
    const uint32_t rev_##L = bitrev32(bits) >> 17;                             \
    const int L = 1 + count_ge16(rev_##L, ll);                                  \
    const int Lc_##L = L <= 15 ? L : 15;                                        \
    const uint32_t e0 = t.ldw(H_LL + 2 * (Lc_##L - 1));                         \
    const uint32_t tc = rev_##L >> (15 - Lc_##L);

// Phase 1 for one block (one lane).  On the device all 32 lanes of the warp call this together (active = false: no block).
template <class Tab, bool LIMS = false, int HDR_WAIT = 512>
BD_HD int huff_phase(const Tab& t, const uint32_t* words, uint64_t byte_off, uint32_t nbytes, uint32_t isize,
                     uint32_t* scratch /* 384 B */, HuffOut ho, uint32_t& n_tok_out, uint32_t& n_seg_out, uint32_t& n_lit_out, bool active = true) {
    unsigned mask = BD_BALLOT(0xFFFFFFFFu, active);
    n_tok_out = 0; n_seg_out = 0; n_lit_out = 0;
    if (!active) return INF_OK;
    uint8_t* lens = reinterpret_cast<uint8_t*>(scratch);
    uint32_t* limpk = scratch + 80;
    BitWin br; br.init(words, byte_off, nbytes, t.fifo_sa);
    HuffPk ll, dd;
#pragma unroll
    for (int i = 0; i < 8; i++) { ll.pk[i] = 0; dd.pk[i] = 0; }
    uint32_t nlit = 0;                              // literals written so far
    uint32_t cur = 0, L0 = 0, L1 = 0, L2 = 0;       // the word / the 16-byte line of the literal stream being filled
    int state = ST_HDR, rc = INF_OK; uint32_t bfinal = 0, stored_rem = 0;
    uint32_t lit_run = 0, ntok = 0, nseg = 0, wait = 0;
    for (;;) {
        BD_STAT(g_inflate_stats.iters++);
        // ---- header round: parked lanes (state == ST_HDR) parse together
        unsigned hm = BD_BALLOT(mask, state == ST_HDR);
        if (hm) {
            wait++;
            if (hm == mask || wait > (uint32_t)HDR_WAIT) {
                wait = 0;
                if (state == ST_HDR) {
                    if (nseg == (uint32_t)MAX_SEG) { rc = INF_FALLBACK; state = ST_DONE; }
                    else {
                        HdrResult2 hr = next_block2(t, br, lens, limpk, ho.lit_tab + nseg * 256u);
                        br = hr.br; rc = hr.rc; state = hr.state; bfinal = hr.bfinal; stored_rem = hr.stored_rem;
                        if (rc) state = ST_DONE;
                        else if (state != ST_DONE) {
                            ho.seg_info[nseg++] = nlit | (hr.raw ? SEG_RAW : 0u);
                            if (state == ST_SYM) {
                                if (LIMS) { t.st_lim(0, limpk); t.st_lim(1, limpk + 8); }
                                else {
#pragma unroll
                                    for (int i = 0; i < 8; i++) { ll.pk[i] = limpk[i]; dd.pk[i] = limpk[8 + i]; }
                                }
                            }
                        }
                    }
                }
            }
        }
        uint32_t lit_d = 0, lit_n = 0;        // literals (ranks) decoded in this iteration, first in the low byte
        int nlL = 0; uint32_t nlt = 0;        // a non-literal symbol decoded in this iteration: its code length (0: none) and code value
        uint32_t used = 0;                    // bits consumed in this iteration
        uint32_t b0 = 0, b1 = 0;              // the 64 bits at the reader's position
        if (state == ST_SYM) {
            if (LIMS) t.ld_lim(0, ll);
            br.window(b0, b1);
            // Three litlen codes, decoded speculatively one behind the other -- no branch between them, the table words of all
            // three are in flight together -- and then chosen: literals are taken while they last (at most three); the first
            // non-literal is taken if it is the first or second code (a match after two literals would need more than the 64
            // bits of the window) and left for the next iteration otherwise.
            BD_LITLEN_PEEK(b0, La, ta, ea)
            BD_LITLEN_PEEK(funnel_r(b0, b1, (uint32_t)Lc_La), Lb, tb, eb)
            BD_LITLEN_PEEK(funnel_r(b0, b1, (uint32_t)(Lc_La + Lc_Lb)), Lc, tc3, ec)
            const bool ok1 = La <= 15, lit1 = ok1 && ta < (ea & 0xFFFFu);
            const bool ok2 = lit1 && Lb <= 15, lit2 = ok2 && tb < (eb & 0xFFFFu);
            const bool lit3 = lit2 && Lc <= 15 && tc3 < (ec & 0xFFFFu);
            if (!ok1) { rc = INF_ERR_CODE; state = ST_DONE; }
            lit_n = (lit1 ? 1u : 0u) + (lit2 ? 1u : 0u) + (lit3 ? 1u : 0u);
            lit_d = ((ta + (ea >> 16)) & 0xFFu) | (((tb + (eb >> 16)) & 0xFFu) << 8) | (((tc3 + (ec >> 16)) & 0xFFu) << 16);
            used = (ok1 ? (uint32_t)La : 0u) + (ok2 ? (uint32_t)Lb : 0u) + (lit3 ? (uint32_t)Lc : 0u);      // an invalid second code is reported when it is the first code of the next iteration
            { const bool m1 = ok1 && !lit1, m2 = ok2 && !lit2; nlL = m1 ? La : (m2 ? Lb : 0); nlt = m1 ? ta : tb; }      // (selects: a branch here made the compiler run the match code below once per case)
        } else if (state == ST_STORED) {
            br.window(b0, b1);
            lit_n = stored_rem < 3u ? stored_rem : 3u;
            lit_d = b0; used = 8 * lit_n;       // (the bytes above lit_n are masked off below)
            stored_rem -= lit_n;
            if (stored_rem == 0) state = bfinal ? ST_DONE : ST_HDR;
        }
        // ---- append the literals to the packed stream
        if (lit_n) {
            BD_STAT(g_inflate_stats.lits += lit_n);
            if (nlit + lit_n > isize) { rc = INF_ERR_OVERRUN; state = ST_DONE; nlL = 0; }
            else {
                const uint32_t k = nlit & 3u;
                const uint64_t tt = (uint64_t)(lit_d & (0xFFFFFFu >> (8 * (3 - lit_n)))) << (8 * k);
                const uint32_t lo = cur | (uint32_t)tt;
                if (k + lit_n >= 4) {
                    const uint32_t w = (nlit >> 2) & 3u;
                    if (w == 3) {
#if defined(__CUDA_ARCH__)
                        *reinterpret_cast<uint4*>(ho.lits + (nlit & ~15u)) = make_uint4(L0, L1, L2, lo);
#else
                        { uint32_t q[4] = {L0, L1, L2, lo}; for (int i = 0; i < 16; i++) ho.lits[(nlit & ~15u) + i] = (uint8_t)(q[i >> 2] >> ((i & 3) * 8)); }
#endif
                    }
                    L0 = w == 0 ? lo : L0; L1 = w == 1 ? lo : L1; L2 = w == 2 ? lo : L2;
                    cur = (uint32_t)(tt >> 32);
                } else cur = lo;
                nlit += lit_n; lit_run += lit_n;
                if (lit_run >= LIT_RUN_MAX) {
                    if (ntok >= ho.tok_cap) { rc = INF_FALLBACK; state = ST_DONE; nlL = 0; }
                    else { ho.tok[ntok++] = lit_run | TOK_NOMATCH; lit_run = 0; }
                }
            }
        }
        // ---- a length / end-of-block symbol: its extra bits, the distance code and its extra bits all lie in the window
        BD_SYNCWARP(mask);       // every lane of the loop is here: the lanes that have a match run the code below together, once
        if (nlL) {
            uint32_t idx = (nlt + t.ldw(H_LL + 2 * (nlL - 1) + 1)) & 0xFFFFu;
            uint32_t s = idx < 32u ? tab_ld8(t, H_NL, (int)idx) : 31u;
            if (s == 0) state = bfinal ? ST_DONE : ST_HDR;
            else if (s > 29u) { rc = INF_ERR_CODE; state = ST_DONE; }
            else {
                if (LIMS) t.ld_lim(1, dd);
                s -= 1;
                uint32_t len, dist = 0; int ds = -1;
                if (s < 8) len = 3 + s;
                else if (s == 28) len = 258;
                else { uint32_t eb2 = (s >> 2) - 1; len = ((4 + (s & 3)) << eb2) + 3 + (win_at(b0, b1, used) & ((1u << eb2) - 1u)); used += eb2; }
                {
                    const uint32_t revd = bitrev32(win_at(b0, b1, used)) >> 17;
                    const int Ld = 1 + count_ge16(revd, dd);
                    if (Ld <= 15) {
                        int didx = (int)(revd >> (15 - Ld)) + (int)(int16_t)tab_ld16(t, H_DD, Ld - 1);
                        if (didx >= 0 && didx < 32) { ds = (int)tab_ld8(t, H_DS, didx); used += (uint32_t)Ld; }
                    }
                }
                if (ds >= 0 && ds <= 29) {
                    if (ds < 4) dist = 1 + (uint32_t)ds;
                    else { uint32_t eb2 = ((uint32_t)ds >> 1) - 1; dist = ((2 + ((uint32_t)ds & 1)) << eb2) + 1 + (win_at(b0, b1, used) & ((1u << eb2) - 1u)); used += eb2; }
                }
                int e = INF_OK;
                if (ds < 0 || ds > 29) e = INF_ERR_CODE;
                else if (br.P + used > br.pend) e = INF_ERR_INPUT;
                else if (ntok >= ho.tok_cap) e = INF_FALLBACK;
                if (e) { rc = e; state = ST_DONE; }
                else {
                    BD_STAT(g_inflate_stats.matches++); BD_STAT(g_inflate_stats.match_bytes += len);
                    ho.tok[ntok++] = lit_run | ((len - 3u) << 8) | ((dist - 1u) << 16);
                    lit_run = 0;
                }
            }
        }
        if (used) { br.advance(used); if (br.overrun()) { rc = INF_ERR_INPUT; state = ST_DONE; } }
        bool cont = state != ST_DONE;
        mask = BD_BALLOT(mask, cont);
        if (!cont) break;
    }
    n_tok_out = ntok; n_seg_out = nseg; n_lit_out = nlit;
    if (rc) return rc;
    if (lit_run) {        // trailing literals
        if (ntok >= ho.tok_cap) return INF_FALLBACK;
        ho.tok[ntok++] = lit_run | TOK_NOMATCH; n_tok_out = ntok;
    }
    if (nlit & 15u) {     // the last, partial line of the literal stream (the area is padded to a multiple of 16 bytes)
        const uint32_t w = (nlit >> 2) & 3u;
        uint32_t q[4] = {w == 0 ? cur : L0, w == 1 ? cur : L1, w == 2 ? cur : L2, w == 3 ? cur : 0u};
#if defined(__CUDA_ARCH__)
        *reinterpret_cast<uint4*>(ho.lits + (nlit & ~15u)) = make_uint4(q[0], q[1], q[2], q[3]);
#else
        for (uint32_t i = 0; i < (nlit & 15u); i++) ho.lits[(nlit & ~15u) + i] = (uint8_t)(q[i >> 2] >> ((i & 3) * 8));
#endif
    }
    return INF_OK;
}
#undef BD_LITLEN_PEEK

// Phase 2, serial restatement (host tests of phase 1's output; the warp version is k1_lz in kernels.cuh): replay the
// tokens; literals come from the packed stream through the table of the deflate block they belong to.
inline int lz_phase_serial(uint8_t* u /* the block's output, isize bytes */, uint32_t isize, const uint32_t* tok, uint32_t n_tok,
                           const uint8_t* lits, uint32_t n_lit, const uint8_t* lit_tab, const uint32_t* seg_info, uint32_t n_seg) {
    uint32_t pos = 0, li = 0, sg = 0;
    for (uint32_t i = 0; i < n_tok; i++) {
        uint32_t tk = tok[i], nl = tk & 0xFFu;
        if (li + nl > n_lit || pos + nl > isize) return INF_ERR_OVERRUN;
        for (uint32_t k = 0; k < nl; k++, li++) {
            while (sg + 1 < n_seg && li >= (seg_info[sg + 1] & 0x7FFFFFFFu)) sg++;
            u[pos++] = (seg_info[sg] & SEG_RAW) ? lits[li] : lit_tab[sg * 256u + lits[li]];
        }
        if (tk & TOK_NOMATCH) continue;
        uint32_t len = ((tk >> 8) & 0xFFu) + 3, dist = ((tk >> 16) & 0x7FFFu) + 1;
        if (dist > pos) return INF_ERR_DIST;
        if (pos + len > isize) return INF_ERR_OVERRUN;
        for (uint32_t k = 0; k < len; k++) u[pos + k] = u[pos + k - dist];
        pos += len;
    }
    if (li != n_lit) return INF_ERR_SHORT;
    return pos == isize ? INF_OK : INF_ERR_SHORT;
}

}  // namespace bdk
