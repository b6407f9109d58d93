// GPU side of the BAM reader (SURVEY 8f row f4; VERDICT r1 item 5): BGZF inflate, record-chain walk, record parse and the
// scatter into the pb_records_t structure-of-arrays — everything htslib's bgzf_read / bam_read1 / sam_itr_next do under
// BAM_handler::get_reads (pepper/modules/src/dataio/bam_handler.cpp:115-135), with only the COMPRESSED bytes crossing PCIe.
//
//   k_bgzf_inflate   one warp per BGZF block (RFC 1951 DEFLATE: stored / fixed / dynamic Huffman blocks).  Lane 0 owns the bit
//                    reader for headers; tables (10-bit literal/length, 8-bit distance, canonical first-code walk for longer
//                    codes) are built by the whole warp.  Symbols: all 32 lanes decode a candidate symbol start speculatively and
//                    the true chain is found with shuffles (spec_symbols); LZ77 copies that depend on the current round are done
//                    by the whole warp (overlapping copies replicate the period: src = pos - dist + i mod dist).
//   k_chain_*        record boundaries: BAM records are chained by their block_size field, a sequential dependency.  The BAI
//                    linear index provides the virtual offset of a record start for every 16 kb window, so one thread per
//                    window start hops its own short chain (count pass, scan, write pass).
//   k_rec_parse      per record: long-CIGAR convention (CG:B,I tag), reference length, htslib overlap rule, sizes.
//   k_rec_scatter    warp per kept record: 4-bit sequence (re-packed when the output nibble offset is odd), qualities, CIGAR.
#pragma once
#include "common.cuh"
#include <stdlib.h>

namespace pb {
namespace bgzf {

struct BlockDesc { int64_t in_off; int32_t in_len; int32_t out_len; int64_t out_off; };

constexpr int LIT_BITS = 10, DIST_BITS = 8;
constexpr int WARPS_PER_CTA = 4;

struct WarpTables {
    uint16_t lit[1 << LIT_BITS];      // (symbol << 4) | code length; 0 = longer than LIT_BITS
    uint16_t dist[1 << DIST_BITS];
    uint16_t code[320];               // canonical code of each symbol (scratch of the table build)
    uint16_t lit_sym[288], dist_sym[32];   // symbols sorted by (length, symbol): canonical slow path
    uint16_t lit_cnt[16], dist_cnt[16];
    uint8_t lens[320];
};

__constant__ uint16_t c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
                                         8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// LSB-first bit reader over 32-bit ALIGNED loads (the payload may start at any byte: the first word is shifted).  Reads may run
// up to 7 bytes past the payload into the next block's header / the buffer padding — consumed positions are checked, not loads.
struct BitReader {
    const uint8_t *p;          // payload start (any alignment)
    const uint32_t *w;         // next aligned word to load
    int64_t end;               // payload length in bytes
    int64_t loaded;            // payload bytes loaded so far (may exceed `end`)
    uint64_t buf;
    int cnt;
    __device__ __forceinline__ void init(const uint8_t *src, int64_t len) {
        p = src; end = len;
        const int mis = (int) ((uintptr_t) src & 3);
        w = reinterpret_cast<const uint32_t *>(src - mis);
        buf = (uint64_t) (*w++ >> (8 * mis));
        cnt = 32 - 8 * mis;
        loaded = 4 - mis;
    }
    __device__ __forceinline__ void refill() {                 // more than 32 valid bits afterwards
        if (cnt <= 32) { buf |= (uint64_t) (*w++) << cnt; cnt += 32; loaded += 4; }
    }
    __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t) buf & ((1u << n) - 1u); }
    __device__ __forceinline__ void skip(int n) { buf >>= n; cnt -= n; }
    __device__ __forceinline__ uint32_t get(int n) { refill(); const uint32_t v = peek(n); skip(n); return v; }
    __device__ __forceinline__ uint32_t get_nofill(int n) { const uint32_t v = peek(n); skip(n); return v; }     // caller guarantees n <= cnt
    __device__ __forceinline__ int64_t consumed() const { return loaded - (cnt >> 3); }                           // whole bytes consumed
    __device__ __forceinline__ bool overrun() const { return consumed() > end; }
    __device__ __forceinline__ int64_t bitpos() const { return loaded * 8 - cnt; }                                // bits consumed so far
    __device__ __forceinline__ void seek_bits(int64_t bit_pos) { seek(bit_pos >> 3); skip((int) (bit_pos & 7)); }
    __device__ __forceinline__ void seek(int64_t byte_pos) {                                                     // restart at a byte position
        const uint8_t *q = p + byte_pos;
        const int mis = (int) ((uintptr_t) q & 3);
        w = reinterpret_cast<const uint32_t *>(q - mis);
        buf = (uint64_t) (*w++ >> (8 * mis));
        cnt = 32 - 8 * mis;
        loaded = byte_pos + 4 - mis;
    }
};

// Builds the primary table + the canonical (count, sorted symbols) arrays for `n` symbols with code lengths lens[0..n).
// Whole warp; returns false when the lengths over-subscribe the code space, and when they leave part of it unused unless
// `lenient` and no code is longer than 1 bit (zlib's inflate_table: a literal/length or distance set may be one 1-bit code
// or empty; a code-length set must be complete).
__device__ bool build_table(const uint8_t *lens, int n, uint16_t *tab, int tab_bits, uint16_t *cnt, uint16_t *sorted, uint16_t *code, bool lenient,
                            int lane) {
    if (lane < 16) cnt[lane] = 0;
    for (int i = lane; i < (1 << tab_bits); i += 32) tab[i] = 0;
    __syncwarp();
    bool ok = true;
    if (lane == 0) {
        for (int s = 0; s < n; s++) cnt[lens[s]]++;
        cnt[0] = 0;
        int left = 1, longest = 0;
        for (int l = 1; l <= 15; l++) { left = (left << 1) - cnt[l]; if (left < 0) ok = false; if (cnt[l]) longest = l; }
        if (left > 0 && !(lenient && longest <= 1)) ok = false;
        // canonical codes + symbols sorted by (length, symbol)
        uint16_t next[16], offs[16];
        uint32_t c = 0;
        uint16_t o = 0;
        for (int l = 1; l <= 15; l++) { c = (c + cnt[l - 1]) << 1; next[l] = (uint16_t) c; offs[l] = o; o += cnt[l]; }
        for (int s = 0; s < n; s++) {
            const int l = lens[s];
            if (l) { code[s] = next[l]++; sorted[offs[l]++] = (uint16_t) s; }
        }
    }
    ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
    __syncwarp();
    if (!ok) return false;
    for (int s = lane; s < n; s += 32) {
        const int l = lens[s];
        if (l && l <= tab_bits) {
            const uint32_t rev = __brev((uint32_t) code[s]) >> (32 - l);       // DEFLATE packs Huffman codes MSB first
            const uint16_t e = (uint16_t) ((s << 4) | l);
            for (uint32_t i = rev; i < (1u << tab_bits); i += 1u << l) tab[i] = e;
        }
    }
    __syncwarp();
    return true;
}

// lane 0 only: one symbol
__device__ __forceinline__ int decode_sym(BitReader &br, const uint16_t *tab, int tab_bits, const uint16_t *cnt, const uint16_t *sorted) {
    br.refill();
    const uint16_t e = tab[br.peek(tab_bits)];
    if (e) { br.skip(e & 15); return e >> 4; }
    // canonical walk for codes longer than the table (RFC 1951 3.2.2): rare
    int code = 0, first = 0, index = 0;
    uint64_t b = br.buf;
    for (int l = 1; l <= 15; l++) {
        code |= (int) (b & 1); b >>= 1;
        const int c = cnt[l];
        if (code - c < first) { br.skip(l); return sorted[index + (code - first)]; }
        index += c; first += c; first <<= 1; code <<= 1;
    }
    return -1;
}

// ---------------------------------------------------------------------------------------------- warp-parallel symbol decode
// The symbol stream of a deflate block is serial (every code length decides where the next code starts), which leaves 31 lanes
// idle in the classic one-decoder-per-warp scheme and makes the kernel instruction-issue bound.  Here all 32 lanes decode
// SPECULATIVELY: lane i decodes the complete symbol (literal, or length + extra + distance + extra) that would start at bit
// bp + i; the true symbol starts are then found by a short walk over the per-lane bit counts (p = 0; p += nbits[p]) done with
// warp shuffles; lanes on the chain own a symbol of this round, store their literal / copy their short match themselves, and
// the rare matches that read bytes produced in the same round (or are long) are copied cooperatively in stream order.
// Roughly 4-5 symbols per round of ~150 warp instructions instead of ~100 instructions per symbol.
enum { K_LIT = 0, K_MATCH = 1, K_EOB = 2, K_BAD = 3, K_SLOW = 4 };

struct SpecTabs { uint16_t len_base[32]; uint16_t dist_base[32]; uint8_t len_extra[32]; uint8_t dist_extra[32]; };

// 64 bits of the payload starting at absolute bit `bit` (aligned 32-bit loads; may read a few bytes past the payload)
__device__ __forceinline__ uint64_t load_window(const uint8_t *p, int64_t bit) {
    const uint64_t a = (uint64_t) (uintptr_t) p * 8ull + (uint64_t) bit;
    const uint32_t *w = reinterpret_cast<const uint32_t *>((uintptr_t) ((a >> 5) << 2));
    const uint32_t sh = (uint32_t) (a & 31);
    const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
    const uint32_t lo = __funnelshift_r(w0, w1, sh), hi = __funnelshift_r(w1, w2, sh);
    return (uint64_t) lo | ((uint64_t) hi << 32);
}

// canonical (first-code) decode of one code from the low bits of `b`; returns the symbol, length in `len` (-1: invalid)
__device__ __forceinline__ int canon_decode(uint64_t b, const uint16_t *cnt, const uint16_t *sorted, int &len) {
    int code = 0, first = 0, index = 0;
    for (int l = 1; l <= 15; l++) {
        code |= (int) (b & 1); b >>= 1;
        const int c = cnt[l];
        if (code - c < first) { len = l; return sorted[index + (code - first)]; }
        index += c; first += c; first <<= 1; code <<= 1;
    }
    len = 1;
    return -1;
}

// one complete symbol from the window; `exact`: codes longer than the lookup tables are resolved (canonical walk), else K_SLOW
__device__ __forceinline__ void decode_full(uint64_t wnd, const WarpTables &T, const SpecTabs &X, bool exact, int &kind, int &nbits, int &olen, int &val, int &dist) {
    kind = K_BAD; nbits = 1; olen = 0; val = 0; dist = 0;
    int l1, sym;
    const uint16_t e = T.lit[(uint32_t) wnd & ((1u << LIT_BITS) - 1u)];
    if (e) { l1 = e & 15; sym = e >> 4; }
    else if (!exact) { kind = K_SLOW; return; }
    else { sym = canon_decode(wnd, T.lit_cnt, T.lit_sym, l1); if (sym < 0) return; }
    if (sym < 256) { kind = K_LIT; nbits = l1; olen = 1; val = sym; return; }
    if (sym == 256) { kind = K_EOB; nbits = l1; return; }
    if (sym > 285) return;
    const int li = sym - 257;
    const int xb = X.len_extra[li];
    const int mlen = X.len_base[li] + (int) ((uint32_t) (wnd >> l1) & ((1u << xb) - 1u));
    const int t = l1 + xb;                                                    // <= 20
    int l2, ds;
    const uint16_t e2 = T.dist[(uint32_t) (wnd >> t) & ((1u << DIST_BITS) - 1u)];
    if (e2) { l2 = e2 & 15; ds = e2 >> 4; }
    else if (!exact) { kind = K_SLOW; return; }
    else { ds = canon_decode(wnd >> t, T.dist_cnt, T.dist_sym, l2); if (ds < 0) return; }
    if (ds > 29) return;
    const int xd = X.dist_extra[ds];
    dist = X.dist_base[ds] + (int) ((uint32_t) (wnd >> (t + l2)) & ((1u << xd) - 1u));
    kind = K_MATCH; nbits = t + l2 + xd; olen = mlen; val = mlen;               // <= 48 bits
}

// decodes symbols from bit position `bp` until the end-of-block code; all 32 lanes.  Returns the error code (0 ok).
__device__ int spec_symbols(const uint8_t *payload, int64_t in_bits, int64_t &bp, uint8_t *dst, int out_len, int &pos, const WarpTables &T, const SpecTabs &X,
                            int lane) {
    for (;;) {
        const uint64_t wnd = load_window(payload, bp + lane);
        int kind, nbits, olen, val, dist;
        decode_full(wnd, T, X, false, kind, nbits, olen, val, dist);
        // ---- the chain of true symbol starts inside [0, 32): uniform walk
        int p = 0, off = 0, myoff = -1, err = 0;
        bool eob = false;
        while (p < 32) {
            int k = __shfl_sync(0xffffffffu, kind, p);
            if (k == K_SLOW) {                                                  // a code longer than the lookup table at a TRUE start: rare
                const uint32_t wl = __shfl_sync(0xffffffffu, (uint32_t) wnd, p), wh = __shfl_sync(0xffffffffu, (uint32_t) (wnd >> 32), p);
                int k2, n2, o2, v2, d2;
                decode_full((uint64_t) wl | ((uint64_t) wh << 32), T, X, true, k2, n2, o2, v2, d2);
                if (lane == p) { kind = k2; nbits = n2; olen = o2; val = v2; dist = d2; }
                k = k2;
            }
            const int n = __shfl_sync(0xffffffffu, nbits, p), o = __shfl_sync(0xffffffffu, olen, p);
            if (k == K_BAD) { err = 3; break; }
            if (lane == p) myoff = off;
            off += o; p += n;
            if (k == K_EOB) { eob = true; break; }
        }
        if (err) return err;
        if (pos + off > out_len) return 4;
        if (bp + p > in_bits) return 7;                                          // a symbol ends past the payload (BitReader::overrun)
        // ---- output: literals and short matches that read only bytes of earlier rounds are written by their own lanes
        const bool mine = myoff >= 0;
        bool coop = false;
        if (mine && kind == K_LIT) dst[pos + myoff] = (uint8_t) val;
        if (mine && kind == K_MATCH) {
            if (dist > pos + myoff) err = 5;
            else if (val <= 8 && dist >= myoff + val) {
                const uint8_t *src = dst + pos + myoff - dist;
#pragma unroll 1
                for (int i = 0; i < val; i++) dst[pos + myoff + i] = src[i];
            } else coop = true;
        }
        if (__any_sync(0xffffffffu, err != 0)) return 5;
        unsigned cm = __ballot_sync(0xffffffffu, coop);
        while (cm) {                                                            // in stream order (= lane order)
            const int j = __ffs(cm) - 1;
            cm &= cm - 1;
            const int o = __shfl_sync(0xffffffffu, myoff, j), l = __shfl_sync(0xffffffffu, val, j), d = __shfl_sync(0xffffffffu, dist, j);
            __syncwarp();                                                       // everything written so far in this round is visible
            const uint8_t *src = dst + pos + o - d;
            if (d >= l) { for (int i = lane; i < l; i += 32) dst[pos + o + i] = src[i]; }
            else { for (int i = lane; i < l; i += 32) dst[pos + o + i] = src[i % d]; }
        }
        pos += off;
        bp += p;
        __syncwarp();                                                           // the next round may read what this one wrote
        if (eob) return 0;
    }
}

// status: 0 ok, 1 bad block type / stored header, 2 bad code lengths, 3 bad symbol, 4 output overrun, 5 distance too far,
//         6 size mismatch, 7 input overrun
template <bool SPEC>
__global__ void __launch_bounds__(32 * WARPS_PER_CTA) k_bgzf_inflate(const uint8_t *__restrict__ comp, const BlockDesc *__restrict__ blocks, int n_blocks,
                                                                     uint8_t *out, int *__restrict__ status) {
    __shared__ WarpTables T_all[WARPS_PER_CTA];
    __shared__ SpecTabs X;
    if (threadIdx.x < 32) {
        X.len_base[threadIdx.x] = threadIdx.x < 29 ? c_len_base[threadIdx.x] : 0; X.len_extra[threadIdx.x] = threadIdx.x < 29 ? c_len_extra[threadIdx.x] : 0;
        X.dist_base[threadIdx.x] = threadIdx.x < 30 ? c_dist_base[threadIdx.x] : 0; X.dist_extra[threadIdx.x] = threadIdx.x < 30 ? c_dist_extra[threadIdx.x] : 0;
    }
    __syncthreads();
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t b = (int64_t) blockIdx.x * WARPS_PER_CTA + wid;
    if (b >= n_blocks) return;
    WarpTables &T = T_all[wid];
    const BlockDesc D = blocks[b];
    uint8_t *dst = out + D.out_off;
    BitReader br;
    br.init(comp + D.in_off, D.in_len);
    int pos = 0, err = 0;
    int last = 0;
    while (!last && !err) {
        int type = 0;
        if (lane == 0) { last = (int) br.get(1); type = (int) br.get(2); }
        last = __shfl_sync(0xffffffffu, last, 0); type = __shfl_sync(0xffffffffu, type, 0);
        if (type == 0) {
            // stored: skip to the byte boundary, LEN / NLEN, raw bytes
            int len = 0;
            int64_t src = 0;
            if (lane == 0) {
                br.skip(br.cnt & 7);
                const uint32_t l = br.get(16), nl = br.get(16);
                if ((l ^ 0xffffu) != nl) err = 1;
                len = (int) l;
                src = br.consumed();                                  // byte position of the next unread input byte
            }
            err = __shfl_sync(0xffffffffu, err, 0); len = __shfl_sync(0xffffffffu, len, 0); src = __shfl_sync(0xffffffffu, src, 0);
            if (!err && (pos + len > D.out_len || src + len > D.in_len)) err = 4;
            if (err) break;
            for (int i = lane; i < len; i += 32) dst[pos + i] = br.p[src + i];
            pos += len;
            if (lane == 0) br.seek(src + len);
            __syncwarp();
            continue;
        }
        if (type == 3) { err = 1; break; }
        int hlit = 288, hdist = 30;
        if (type == 1) {
            for (int s = lane; s < 288; s += 32) T.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
            T.lens[288 + lane] = 5;                                     // distances 30 / 31 complete the code; decoding them is an error
            __syncwarp();
        } else {
            // dynamic: HLIT, HDIST, HCLEN, the code-length code, then the literal/length + distance code lengths
            int hclen = 0;
            if (lane == 0) { hlit = (int) br.get(5) + 257; hdist = (int) br.get(5) + 1; hclen = (int) br.get(4) + 4; }
            hlit = __shfl_sync(0xffffffffu, hlit, 0); hdist = __shfl_sync(0xffffffffu, hdist, 0);
            if (hlit > 286 || hdist > 30) { err = 2; break; }
            if (lane < 19) T.lens[lane] = 0;
            __syncwarp();
            if (lane == 0) for (int i = 0; i < hclen; i++) T.lens[c_clen_order[i]] = (uint8_t) br.get(3);
            __syncwarp();
            if (!build_table(T.lens, 19, T.dist, 7, T.dist_cnt, T.dist_sym, T.code, false, lane)) { err = 2; break; }
            if (lane == 0) {
                uint8_t tmp[320];
                int i = 0;
                const int total = hlit + hdist;
                while (i < total && !err) {
                    const int s = decode_sym(br, T.dist, 7, T.dist_cnt, T.dist_sym);
                    if (s < 0) { err = 2; break; }
                    if (s < 16) { tmp[i++] = (uint8_t) s; continue; }
                    int rep, val = 0;
                    if (s == 16) { if (i == 0) { err = 2; break; } val = tmp[i - 1]; rep = 3 + (int) br.get(2); }
                    else if (s == 17) rep = 3 + (int) br.get(3);
                    else rep = 11 + (int) br.get(7);
                    if (i + rep > total) { err = 2; break; }
                    while (rep--) tmp[i++] = (uint8_t) val;
                }
                if (!err) {
                    for (int k = 0; k < hlit; k++) T.lens[k] = tmp[k];
                    for (int k = hlit; k < 288; k++) T.lens[k] = 0;
                    for (int k = 0; k < hdist; k++) T.lens[288 + k] = tmp[hlit + k];
                    for (int k = hdist; k < 32; k++) T.lens[288 + k] = 0;
                    if (T.lens[256] == 0) err = 2;                      // no end-of-block code
                }
            }
            err = __shfl_sync(0xffffffffu, err, 0);
            if (err) break;
            __syncwarp();
        }
        if (!build_table(T.lens, 288, T.lit, LIT_BITS, T.lit_cnt, T.lit_sym, T.code, true, lane)) { err = 2; break; }
        if (!build_table(T.lens + 288, 32, T.dist, DIST_BITS, T.dist_cnt, T.dist_sym, T.code, true, lane)) { err = 2; break; }
        if (SPEC) {
            // ---- warp-parallel speculative decode (above); lane 0's bit reader is re-synchronised at the end-of-block position
            int64_t bp = 0;
            if (lane == 0) bp = br.bitpos();
            bp = __shfl_sync(0xffffffffu, bp, 0);
            pos = __shfl_sync(0xffffffffu, pos, 0);
            err = spec_symbols(br.p, (int64_t) D.in_len * 8, bp, dst, D.out_len, pos, T, X, lane);
            if (err) break;
            if (lane == 0) br.seek_bits(bp);
            continue;
        }
        // ---- symbols: lane 0 decodes (writing literals itself) up to the next match / end of block, the warp performs the copy.
        //      One packed broadcast per match: bits 0-15 distance (1..32768), 16-24 length, 28-30 error, bit 31 end of block.
        for (;;) {
            uint32_t msg = 0;
            if (lane == 0) {
                for (;;) {
                    const int s = decode_sym(br, T.lit, LIT_BITS, T.lit_cnt, T.lit_sym);          // refills: > 32 bits before, >= 18 after
                    if (s < 256) {
                        if (s < 0) { err = 3; break; }
                        if (pos >= D.out_len) { err = 4; break; }
                        dst[pos++] = (uint8_t) s;
                        continue;
                    }
                    if (s == 256) { msg = 0x80000000u; break; }
                    if (s > 285) { err = 3; break; }
                    const int li = s - 257;
                    const int mlen = c_len_base[li] + (int) br.get_nofill(c_len_extra[li]);       // <= 5 extra bits: still in the buffer
                    const int ds = decode_sym(br, T.dist, DIST_BITS, T.dist_cnt, T.dist_sym);      // refills again: > 32 bits before
                    if (ds < 0 || ds > 29) { err = 3; break; }
                    const int mdist = c_dist_base[ds] + (int) br.get_nofill(c_dist_extra[ds]);    // 15 + 13 bits <= 32
                    msg = (uint32_t) (mdist & 0xffff) | ((uint32_t) mlen << 16);
                    break;
                }
                if (br.overrun()) err = 7;
                msg |= (uint32_t) err << 28;
            }
            msg = __shfl_sync(0xffffffffu, msg, 0);
            pos = __shfl_sync(0xffffffffu, pos, 0);
            err = (int) ((msg >> 28) & 7u);
            if (err) break;
            if (msg >> 31) break;                                       // end of this deflate block
            const int mlen = (int) ((msg >> 16) & 0x1ffu);
            const int mdist = (msg & 0xffffu) ? (int) (msg & 0xffffu) : 65536;     // 32768 fits; 0 cannot occur (bases start at 1)
            if (mdist > pos) { err = 5; break; }
            if (pos + mlen > D.out_len) { err = 4; break; }
            __syncwarp();                                               // earlier stores of this warp (literals, previous copy) are visible
            const uint8_t *src = dst + pos - mdist;
            if (mdist >= mlen) {
                for (int i = lane; i < mlen; i += 32) dst[pos + i] = src[i];
            } else {
                for (int i = lane; i < mlen; i += 32) dst[pos + i] = src[i % mdist];
            }
            pos += mlen;
        }
    }
    if (!err && pos != D.out_len) err = 6;
    if (lane == 0) status[b] = err;
}

// PB_INFLATE_SPEC=0 selects the one-decoder-per-warp symbol loop (cross-check); default: the warp-parallel speculative decode
static inline int launch_inflate(const uint8_t *comp, const BlockDesc *blocks, int64_t n_blocks, uint8_t *out, int *status, cudaStream_t st) {
    static const bool spec = !(getenv("PB_INFLATE_SPEC") && atoi(getenv("PB_INFLATE_SPEC")) == 0);
    const unsigned grid = (unsigned) ceil_div(n_blocks, WARPS_PER_CTA);
    if (spec) k_bgzf_inflate<true><<<grid, 32 * WARPS_PER_CTA, 0, st>>>(comp, blocks, (int) n_blocks, out, status);
    else k_bgzf_inflate<false><<<grid, 32 * WARPS_PER_CTA, 0, st>>>(comp, blocks, (int) n_blocks, out, status);
    PB_CUDA(cudaGetLastError());
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------------ record chains
__device__ __forceinline__ uint32_t ld_u32(const uint8_t *p) { return (uint32_t) p[0] | ((uint32_t) p[1] << 8) | ((uint32_t) p[2] << 16) | ((uint32_t) p[3] << 24); }
__device__ __forceinline__ uint32_t ld_u16(const uint8_t *p) { return (uint32_t) p[0] | ((uint32_t) p[1] << 8); }

// thread per chain start: hop record to record from starts[i] until starts[i + 1] (or `limit`); WRITE = 0 counts, 1 writes offsets
// (starts[i], stops[i]): stops[i] = the next known record start of the same chunk group, or the group's end
template <int WRITE>
__global__ void k_chain(const uint8_t *__restrict__ u, const int64_t *__restrict__ starts, const int64_t *__restrict__ stops, int n_starts,
                        int32_t *__restrict__ counts, const int64_t *__restrict__ base, int64_t *__restrict__ rec_off, int *__restrict__ err) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_starts) return;
    int64_t p = starts[i];
    const int64_t stop = stops[i];
    int64_t k = WRITE ? base[i] : 0;
    int32_t n = 0;
    while (p + 4 <= stop) {
        const uint32_t bs = ld_u32(u + p);
        if (bs < 32 || p + 4 + (int64_t) bs > stop) { atomicExch(err, 1); break; }     // a record runs over the next known record start / its chunk
        if (WRITE) rec_off[k++] = p;
        n++;
        p += 4 + (int64_t) bs;
    }
    if (!WRITE) counts[i] = n;
}

struct RecInfo { int64_t cigar_pos; int32_t n_cigar, l_seq; int32_t pos; uint8_t keep; };

// thread per record: tid / position window, long-CIGAR convention (SAMv1 4.2.2), reference length, htslib overlap rule
__global__ void k_rec_parse(const uint8_t *__restrict__ u, const int64_t *__restrict__ rec_off, int64_t n_rec, int tid, int64_t beg, int64_t end,
                            RecInfo *__restrict__ info, int32_t *__restrict__ keep32, int32_t *__restrict__ lseq32, int32_t *__restrict__ ncig32,
                            int *__restrict__ err) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_rec) return;
    const int64_t p = rec_off[i];
    const uint32_t bs = ld_u32(u + p);
    const uint8_t *r = u + p + 4;
    const int32_t rtid = (int32_t) ld_u32(r), pos = (int32_t) ld_u32(r + 4);
    const uint32_t l_name = r[8], n_cig = ld_u16(r + 12), l_seq = ld_u32(r + 16);
    RecInfo I;
    I.pos = pos; I.l_seq = (int32_t) l_seq; I.keep = 0; I.n_cigar = 0; I.cigar_pos = 0;
    if (32ull + l_name + 4ull * n_cig + (l_seq + 1) / 2 + l_seq > bs) { atomicExch(err, 3); info[i] = I; keep32[i] = 0; lseq32[i] = 0; ncig32[i] = 0; return; }
    if (rtid == tid && pos < end) {
        const uint8_t *cig = r + 32 + l_name;
        uint32_t n_cigar = n_cig;
        const uint8_t *cigar = cig;
        if (n_cig == 2 && (ld_u32(cig) & 15) == 4 && (ld_u32(cig) >> 4) == l_seq && (ld_u32(cig + 4) & 15) == 3) {
            const uint8_t *a = cig + 8 + (l_seq + 1) / 2 + l_seq, *ae = r + bs;
            while (a + 3 <= ae) {
                const char t0 = (char) a[0], t1 = (char) a[1], ty = (char) a[2];
                a += 3;
                size_t sz = 0;
                if (ty == 'A' || ty == 'c' || ty == 'C') sz = 1;
                else if (ty == 's' || ty == 'S') sz = 2;
                else if (ty == 'i' || ty == 'I' || ty == 'f') sz = 4;
                else if (ty == 'Z' || ty == 'H') { while (a + sz < ae && a[sz]) sz++; sz++; }
                else if (ty == 'B') {
                    if (a + 5 > ae) break;
                    const char st = (char) a[0];
                    const uint32_t cnt = ld_u32(a + 1);
                    const size_t es = (st == 'c' || st == 'C') ? 1 : (st == 's' || st == 'S') ? 2 : 4;
                    if (t0 == 'C' && t1 == 'G' && st == 'I' && a + 5 + 4ull * cnt <= ae) { n_cigar = cnt; cigar = a + 5; }
                    sz = 5 + es * cnt;
                } else break;
                a += sz;
            }
        }
        int64_t rlen = 0;
        for (uint32_t k = 0; k < n_cigar; k++) {
            const uint32_t c = ld_u32(cigar + 4 * k);
            const int op = (int) (c & 15);
            if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rlen += c >> 4;
        }
        if (n_cigar == 0) rlen = 1;
        I.n_cigar = (int32_t) n_cigar; I.cigar_pos = (int64_t) (cigar - u);
        I.keep = ((int64_t) pos + rlen > beg) ? 1 : 0;
    }
    info[i] = I;
    keep32[i] = I.keep;
    lseq32[i] = I.keep ? I.l_seq : 0;
    ncig32[i] = I.keep ? I.n_cigar : 0;
}

__device__ __forceinline__ int nib(const uint8_t *s, int64_t k) { return (k & 1) ? (s[k >> 1] & 15) : (s[k >> 1] >> 4); }

// warp per kept record: out index j = keep_off[i]; sequence nibbles at so[j] (contiguous packing across records: the byte shared
// with the previous record is written by the LATER record, as pb_bam_fetch does), qualities, CIGAR words, pos / flag / mapq
__global__ void __launch_bounds__(256) k_rec_scatter(const uint8_t *__restrict__ u, const int64_t *__restrict__ rec_off, const RecInfo *__restrict__ info,
                                                     const int64_t *__restrict__ keep_off, const int64_t *__restrict__ so_all, const int64_t *__restrict__ co_all,
                                                     int64_t n_rec, int64_t *__restrict__ o_pos, int64_t *__restrict__ o_seq_off, int64_t *__restrict__ o_cigar_off,
                                                     uint16_t *__restrict__ o_flag, uint8_t *__restrict__ o_mapq, uint8_t *__restrict__ o_seq,
                                                     uint8_t *__restrict__ o_qual, uint32_t *__restrict__ o_cigar) {
    const int64_t i = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n_rec) return;
    const RecInfo I = info[i];
    if (!I.keep) return;
    const int64_t j = keep_off[i], so = so_all[i], co = co_all[i];
    const uint8_t *r = u + rec_off[i] + 4;
    const uint8_t *s = r + 32 + r[8] + 4 * (size_t) ld_u16(r + 12);
    const int64_t l = I.l_seq;
    if (lane == 0) { o_pos[j] = I.pos; o_seq_off[j] = so; o_cigar_off[j] = co; o_flag[j] = (uint16_t) ld_u16(r + 14); o_mapq[j] = r[9]; }
    const uint8_t *cg = u + I.cigar_pos;
    for (int k = lane; k < I.n_cigar; k += 32) o_cigar[co + k] = ld_u32(cg + 4 * k);
    const uint8_t *q = s + (l + 1) / 2;
    for (int64_t k = lane; k < l; k += 32) o_qual[so + k] = q[k];
    // output bytes [ceil(so/2) .. floor((so+l)/2)) are wholly this record's; a leading shared byte (so odd) is written here too with the
    // previous record's last nibble, fetched from ITS source (the previous kept record that has bases)
    if (!(so & 1)) {
        for (int64_t B = lane; B < (l >> 1); B += 32) o_seq[(so >> 1) + B] = s[B];
    } else if (l > 0) {
        for (int64_t B = ((so + 1) >> 1) + lane; B < ((so + l) >> 1); B += 32) {
            const int64_t k = 2 * B - so;
            o_seq[B] = (uint8_t) (nib(s, k) << 4 | nib(s, k + 1));
        }
        if (lane == 0) {
            int64_t pv = i - 1;
            while (!(info[pv].keep && info[pv].l_seq > 0)) pv--;         // so odd => an earlier kept record has bases
            const uint8_t *rp = u + rec_off[pv] + 4;
            const uint8_t *sp = rp + 32 + rp[8] + 4 * (size_t) ld_u16(rp + 12);
            o_seq[so >> 1] = (uint8_t) (nib(sp, info[pv].l_seq - 1) << 4 | nib(s, 0));
        }
    }
    // a trailing half byte of the LAST base of the batch is written by k_rec_tail
}

// the trailing half byte when the total base count is odd: last kept record with bases
__global__ void k_rec_tail(const uint8_t *__restrict__ u, const int64_t *__restrict__ rec_off, const RecInfo *__restrict__ info, int64_t n_rec, int64_t nb,
                           uint8_t *__restrict__ o_seq) {
    if (threadIdx.x || blockIdx.x || !(nb & 1)) return;
    int64_t last = n_rec - 1;
    while (last >= 0 && !(info[last].keep && info[last].l_seq > 0)) last--;
    if (last < 0) return;
    const uint8_t *r = u + rec_off[last] + 4;
    const uint8_t *s = r + 32 + r[8] + 4 * (size_t) ld_u16(r + 12);
    o_seq[nb >> 1] = (uint8_t) (nib(s, info[last].l_seq - 1) << 4);
}

}  // namespace bgzf
}  // namespace pb
