// BGZF compression on the GPU: each member (<= 65,280 payload bytes, SAMv1 §4.1) becomes one complete gzip member with a
// BSIZE extra field, raw DEFLATE (RFC 1951), CRC32 and ISIZE.  One CTA per member, the payload in shared memory:
//
//   CRC32 per thread chunk, combined by multiplication with x^(8 len) mod P
//   -> hash chains: a 3-byte hash per position; each position's predecessor of the same hash, found by a backward scan of its
//      512-position window or, failing that, the table of the last position per hash before the window
//   -> longest match per position (every position at once): up to MATCH_CHAIN candidates of its chain within 32 KiB of the
//      member, so the window never reaches outside the member
//   -> greedy parse walked by one thread over tiles of the per-position matches; symbol histograms on the way
//   -> dynamic Huffman codes (15-bit limit; 7 for the code-length code) built by one thread; a code over the limit is rebuilt
//      from halved counts
//   -> bit offsets of the tokens from a block prefix sum, packed in parallel with shared atomicOr
//   -> stored blocks instead when the dynamic block would be larger than the payload.
// Output: one 64 KiB slot per member, then a compacting copy to the caller's buffer.
#include "common.cuh"
#include <cub/block/block_scan.cuh>
#include <vector>

namespace pb {

constexpr int DF_THREADS = 512;
constexpr int DF_PAYLOAD = 65280;                  // BGZF_PAYLOAD: the largest member payload
constexpr int DF_SLOT = 65536;                     // a BGZF member is at most 64 KiB
constexpr int DF_HASH_BITS = 13;
constexpr int DF_HASH = 1 << DF_HASH_BITS;
constexpr int DF_WINDOW = 32768;
constexpr int DF_MAX_MATCH = 258;
constexpr int MATCH_CHAIN = 8;
constexpr int DF_TILE = 8192;                      // parse tile: per-position matches staged in shared memory
constexpr int DF_BATCH = 1024;                     // members per launch (global scratch: 256 KiB + 64 KiB each)
constexpr int DF_SMEM = 65536 + 131072 + DF_HASH * 2;

__constant__ uint16_t c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                        131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                         2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ __forceinline__ int len_code(int len) {        // 0..28 (symbol 257 + code)
    if (len == 258) return 28;
    const int l = len - 3;
    if (l < 8) return l;
    const int k = 31 - __clz(l);
    return 4 * (k - 1) + ((l >> (k - 2)) & 3);
}
__device__ __forceinline__ int dist_code(int d) {         // 0..29
    if (d <= 4) return d - 1;
    const int k = 31 - __clz(d - 1);
    return 2 * k + (((d - 1) >> (k - 1)) & 1);
}
__device__ __forceinline__ int dist_extra(int c) { return c < 4 ? 0 : c / 2 - 1; }

// CRC-32 (reflected, polynomial 0xEDB88320) helpers: a * b mod P, and x^(8 n) mod P
__device__ uint32_t crc_multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}
__device__ uint32_t crc_x8n(uint64_t n) {
    uint32_t p = 1u << 31, sq = 1u << 30;                 // x^0, x^1
    n *= 8;
    while (n) {
        if (n & 1) p = crc_multmodp(sq, p);
        sq = crc_multmodp(sq, sq);
        n >>= 1;
    }
    return p;
}

// Huffman code lengths for freq[0..n) limited to `limit` bits (one thread).  Symbols with freq 0 get length 0; the caller
// guarantees at least two non-zero counts, so the code is complete.  Over the limit: halve the counts and rebuild.
struct HuffWork {
    uint16_t sym[320];
    uint32_t w[640];
    int16_t parent[640];
    uint16_t depth[640];
};
__device__ void huff_lengths(const uint32_t *freq_in, int n, int limit, uint8_t *len, HuffWork &H) {
    uint32_t scale = 0;
    for (;;) {
        int m = 0;
        for (int s = 0; s < n; s++) {
            len[s] = 0;
            if (freq_in[s]) {
                // insertion sort by (weight, symbol)
                const uint32_t f = max(1u, freq_in[s] >> scale);
                int k = m++;
                while (k > 0 && H.w[k - 1] > f) { H.w[k] = H.w[k - 1]; H.sym[k] = H.sym[k - 1]; k--; }
                H.w[k] = f; H.sym[k] = (uint16_t) s;
            }
        }
        // two-queue merge: leaves 0..m-1 (sorted), internal nodes m.. created in non-decreasing weight order
        int li = 0, ii = m, nn = m;
        for (int t = 0; t < m - 1; t++) {
            int pick[2];
            for (int c = 0; c < 2; c++) {
                if (li < m && (ii >= nn || H.w[li] <= H.w[ii])) pick[c] = li++;
                else pick[c] = ii++;
            }
            H.w[nn] = H.w[pick[0]] + H.w[pick[1]];
            H.parent[pick[0]] = (int16_t) nn; H.parent[pick[1]] = (int16_t) nn;
            nn++;
        }
        H.depth[nn - 1] = 0;
        int maxd = 0;
        for (int v = nn - 2; v >= 0; v--) {
            H.depth[v] = (uint16_t) (H.depth[H.parent[v]] + 1);
            if (v < m) maxd = max(maxd, (int) H.depth[v]);
        }
        if (maxd <= limit) {
            for (int k = 0; k < m; k++) len[H.sym[k]] = H.depth[k];
            return;
        }
        scale++;
    }
}

// canonical codes, bit-reversed for LSB-first packing
__device__ void huff_codes(const uint8_t *len, int n, uint16_t *code) {
    int bl_count[16] = {0}, next[16];
    for (int s = 0; s < n; s++) bl_count[len[s]]++;
    bl_count[0] = 0;
    int c = 0;
    for (int b = 1; b < 16; b++) { c = (c + bl_count[b - 1]) << 1; next[b] = c; }
    for (int s = 0; s < n; s++) {
        const int l = len[s];
        if (!l) { code[s] = 0; continue; }
        const uint32_t v = (uint32_t) next[l]++;
        code[s] = (uint16_t) (__brev(v) >> (32 - l));
    }
}

struct DfShared {
    uint32_t crc_table[256];
    uint32_t chunk_crc[DF_THREADS];
    uint16_t wh[DF_THREADS];
    uint8_t succ[DF_THREADS];
    uint32_t f_ll[286], f_d[30], f_cl[19];
    uint8_t l_ll[286], l_d[30], l_cl[19];
    uint16_t c_ll[286], c_d[30], c_cl[19];
    uint16_t cl_sym[320];                          // run-length coded code lengths: symbol | extra << 5
    HuffWork H;
    int n_tok, parse_pos, n_cl, hlit, hdist, hclen, stored;
    int64_t total_bits;
    uint32_t crc;
};

__device__ __forceinline__ uint32_t hash3(const uint8_t *d, int i) {
    const uint32_t v = (uint32_t) d[i] | ((uint32_t) d[i + 1] << 8) | ((uint32_t) d[i + 2] << 16);
    return (v * 2654435761u) >> (32 - DF_HASH_BITS);
}

__device__ __forceinline__ void put_bits(uint32_t *words, int64_t off, uint32_t v, int n) {     // n <= 32, v < 2^n
    if (!n) return;
    const uint64_t x = (uint64_t) v << (off & 31);
    atomicOr(&words[off >> 5], (uint32_t) x);
    if ((off & 31) + n > 32) atomicOr(&words[(off >> 5) + 1], (uint32_t) (x >> 32));
}

__global__ void __launch_bounds__(DF_THREADS, 1)
k_bgzf_deflate(const uint8_t *__restrict__ payload, const int64_t *__restrict__ member_off, uint32_t *__restrict__ scratch,
               uint8_t *__restrict__ slots, int64_t *__restrict__ out_bytes) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ DfShared S;
    uint8_t *data = smem;                                              // [65536] payload
    uint16_t *prev = reinterpret_cast<uint16_t *>(smem + 65536);      // [65536] chain: same-hash predecessor + 1 (0 = none)
    uint32_t *tile = reinterpret_cast<uint32_t *>(smem + 65536);      // reuses prev: parse tile, then the output bit buffer
    uint16_t *head = reinterpret_cast<uint16_t *>(smem + 65536 + 131072);
    const int t = threadIdx.x;
    const int m = blockIdx.x;
    const int64_t base = member_off[m];
    const int n = (int) (member_off[m + 1] - base);
    uint32_t *mi = scratch + (size_t) m * DF_PAYLOAD;
    uint8_t *slot = slots + (size_t) m * DF_SLOT;

    for (int i = t; i < n; i += DF_THREADS) data[i] = payload[base + i];
    for (int i = n + t; i < n + 4 && i < 65536; i += DF_THREADS) data[i] = 0;
    for (int i = t; i < DF_HASH; i += DF_THREADS) head[i] = 0;
    for (int i = t; i < 256; i += DF_THREADS) {
        uint32_t c = (uint32_t) i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0xedb88320u : c >> 1;
        S.crc_table[i] = c;
    }
    for (int i = t; i < 286; i += DF_THREADS) S.f_ll[i] = 0;
    if (t < 30) S.f_d[t] = 0;
    __syncthreads();

    // ---- CRC32: one chunk per thread, combined in order
    const int chunk = (n + DF_THREADS - 1) / DF_THREADS;
    {
        const int a = min(n, t * chunk), b = min(n, a + chunk);
        uint32_t c = 0xffffffffu;
        for (int i = a; i < b; i++) c = S.crc_table[(c ^ data[i]) & 255] ^ (c >> 8);
        S.chunk_crc[t] = c ^ 0xffffffffu;
    }
    __syncthreads();
    if (t == 0) {
        uint32_t crc = 0;                                              // CRC of the empty string
        if (n > 0) {
            const uint32_t shift = crc_x8n((uint64_t) chunk);
            const int chunks = (n + chunk - 1) / chunk;
            for (int k = 0; k < chunks; k++) {
                const int len = min(chunk, n - k * chunk);
                crc = crc_multmodp(len == chunk ? shift : crc_x8n((uint64_t) len), crc) ^ S.chunk_crc[k];
            }
        }
        S.crc = crc;
    }

    // ---- hash chains, window by window
    for (int w0 = 0; w0 < n; w0 += DF_THREADS) {
        const int i = w0 + t;
        const bool has = i + 2 < n;
        const uint32_t h = has ? hash3(data, i) : 0xffffu;
        S.wh[t] = (uint16_t) h;
        S.succ[t] = 0;
        __syncthreads();
        if (has) {
            int p = 0;
            for (int s = t - 1; s >= 0; s--)
                if (S.wh[s] == h) { p = w0 + s + 1; S.succ[s] = 1; break; }
            if (!p) p = head[h];
            prev[i] = (uint16_t) p;
        } else if (i < n) {
            prev[i] = 0;
        }
        __syncthreads();
        if (has && !S.succ[t]) head[h] = (uint16_t) (i + 1);           // the last position of this hash in the window
        __syncthreads();
    }

    // ---- longest match per position
    for (int i = t; i < n; i += DF_THREADS) {
        int best = 0, bdist = 0;
        const int maxl = min(DF_MAX_MATCH, n - i);
        if (maxl >= 3) {
            int c = prev[i];
            for (int k = 0; k < MATCH_CHAIN && c; k++) {
                const int j = c - 1;
                if (i - j > DF_WINDOW) break;
                if (data[j + best] == data[i + best]) {
                    int l = 0;
                    while (l < maxl && data[j + l] == data[i + l]) l++;
                    if (l > best) { best = l; bdist = i - j; if (l == maxl) break; }
                }
                c = prev[j];
            }
        }
        mi[i] = best >= 3 ? ((uint32_t) best << 16) | (uint32_t) bdist : 0u;
    }
    __syncthreads();

    // ---- greedy parse (one thread), tokens written over mi: literal = byte, match = len << 16 | dist
    if (t == 0) { S.parse_pos = 0; S.n_tok = 0; }
    __syncthreads();
    while (S.parse_pos < n) {
        const int t0 = S.parse_pos;
        const int tn = min(DF_TILE, n - t0);
        for (int k = t; k < tn; k += DF_THREADS) tile[k] = mi[t0 + k];
        __syncthreads();
        if (t == 0) {
            int i = t0, nt = S.n_tok;
            while (i < t0 + tn) {
                const uint32_t v = tile[i - t0];
                if (v) {
                    const int len = (int) (v >> 16), d = (int) (v & 0xffff);
                    mi[nt++] = v;
                    S.f_ll[257 + len_code(len)]++;
                    S.f_d[dist_code(d)]++;
                    i += len;
                } else {
                    mi[nt++] = data[i];
                    S.f_ll[data[i]]++;
                    i++;
                }
            }
            S.parse_pos = i; S.n_tok = nt;
        }
        __syncthreads();
    }
    const int n_tok = S.n_tok;

    // ---- Huffman codes, header, size (one thread)
    if (t == 0) {
        S.f_ll[256] = 1;
        int nzd = 0;
        for (int s = 0; s < 30; s++) nzd += S.f_d[s] != 0;
        if (nzd < 2) { S.f_d[0] = max(S.f_d[0], 1u); S.f_d[1] = max(S.f_d[1], 1u); }
        int nzl = 0;
        for (int s = 0; s < 286; s++) nzl += S.f_ll[s] != 0;
        if (nzl < 2) S.f_ll[S.f_ll[0] ? 1 : 0] = 1;
        huff_lengths(S.f_ll, 286, 15, S.l_ll, S.H);
        huff_lengths(S.f_d, 30, 15, S.l_d, S.H);
        int hlit = 286, hdist = 30;
        while (hlit > 257 && !S.l_ll[hlit - 1]) hlit--;
        while (hdist > 1 && !S.l_d[hdist - 1]) hdist--;
        // run-length code the lengths (RFC 1951 3.2.7): 16 = repeat previous 3-6, 17 = zeros 3-10, 18 = zeros 11-138
        uint8_t all[316];
        for (int s = 0; s < hlit; s++) all[s] = S.l_ll[s];
        for (int s = 0; s < hdist; s++) all[hlit + s] = S.l_d[s];
        const int tot = hlit + hdist;
        for (int s = 0; s < 19; s++) S.f_cl[s] = 0;
        int nc = 0;
        for (int s = 0; s < tot;) {
            const int v = all[s];
            int r = 1;
            while (s + r < tot && all[s + r] == v) r++;
            if (v == 0 && r >= 3) {
                const int k = min(r, 138);
                if (k >= 11) { S.cl_sym[nc++] = (uint16_t) (18 | ((k - 11) << 5)); S.f_cl[18]++; }
                else { S.cl_sym[nc++] = (uint16_t) (17 | ((k - 3) << 5)); S.f_cl[17]++; }
                s += k;
            } else if (v != 0 && r >= 4) {
                S.cl_sym[nc++] = (uint16_t) v; S.f_cl[v]++;
                const int k = min(r - 1, 6);
                S.cl_sym[nc++] = (uint16_t) (16 | ((k - 3) << 5)); S.f_cl[16]++;
                s += 1 + k;
            } else {
                S.cl_sym[nc++] = (uint16_t) v; S.f_cl[v]++;
                s++;
            }
        }
        int nzc = 0;
        for (int s = 0; s < 19; s++) nzc += S.f_cl[s] != 0;
        if (nzc < 2) S.f_cl[S.f_cl[0] ? 1 : 0] = max(S.f_cl[S.f_cl[0] ? 1 : 0], 1u);
        huff_lengths(S.f_cl, 19, 7, S.l_cl, S.H);
        int hclen = 19;
        while (hclen > 4 && !S.l_cl[c_cl_order[hclen - 1]]) hclen--;
        huff_codes(S.l_ll, 286, S.c_ll);
        huff_codes(S.l_d, 30, S.c_d);
        huff_codes(S.l_cl, 19, S.c_cl);
        int64_t bits = 3 + 5 + 5 + 4 + 3 * hclen;
        for (int k = 0; k < nc; k++) {
            const int s = S.cl_sym[k] & 31;
            bits += S.l_cl[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
        }
        // (a dist / literal count forced to 1 above adds a few bits that are never written: the estimate errs towards stored)
        for (int s = 0; s < 286; s++) bits += (int64_t) S.f_ll[s] * (S.l_ll[s] + (s > 256 ? c_len_extra[s - 257] : 0));
        for (int s = 0; s < 30; s++) bits += (int64_t) S.f_d[s] * (S.l_d[s] + dist_extra(s));
        S.total_bits = bits;
        S.n_cl = nc; S.hlit = hlit; S.hdist = hdist; S.hclen = hclen;
        S.stored = n == 0 || (bits + 7) / 8 >= (int64_t) n + 5;
    }
    __syncthreads();

    int64_t dbytes;
    uint8_t *dst = slot + 18;
    if (S.stored) {
        // one stored block: BFINAL = 1, BTYPE = 00, byte-aligned LEN / NLEN
        if (t == 0) {
            dst[0] = 1;
            dst[1] = (uint8_t) n; dst[2] = (uint8_t) (n >> 8);
            dst[3] = (uint8_t) ~n; dst[4] = (uint8_t) (~n >> 8);
        }
        for (int i = t; i < n; i += DF_THREADS) dst[5 + i] = data[i];
        dbytes = 5 + n;
    } else {
        uint32_t *words = tile;
        for (int k = t; k < 65536 / 4 + 1; k += DF_THREADS) words[k] = 0;
        __syncthreads();
        __shared__ int64_t hdr_bits;
        if (t == 0) {
            int64_t o = 0;
            put_bits(words, o, 1 | (2 << 1), 3); o += 3;                   // BFINAL, BTYPE = 10 (dynamic)
            put_bits(words, o, S.hlit - 257, 5); o += 5;
            put_bits(words, o, S.hdist - 1, 5); o += 5;
            put_bits(words, o, S.hclen - 4, 4); o += 4;
            for (int k = 0; k < S.hclen; k++) { put_bits(words, o, S.l_cl[c_cl_order[k]], 3); o += 3; }
            for (int k = 0; k < S.n_cl; k++) {
                const int s = S.cl_sym[k] & 31, x = S.cl_sym[k] >> 5;
                put_bits(words, o, S.c_cl[s], S.l_cl[s]); o += S.l_cl[s];
                const int eb = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
                put_bits(words, o, (uint32_t) x, eb); o += eb;
            }
            hdr_bits = o;
        }
        __syncthreads();
        // tokens: bit length -> block exclusive scan -> parallel packing
        typedef cub::BlockScan<int64_t, DF_THREADS> Scan;
        __shared__ typename Scan::TempStorage scan_tmp;
        __shared__ int64_t carry;
        if (t == 0) carry = hdr_bits;
        __syncthreads();
        for (int k0 = 0; k0 < n_tok; k0 += DF_THREADS) {
            const int k = k0 + t;
            uint32_t v = 0;
            int nb = 0, lc = 0, dc = 0, len = 0, d = 0;
            if (k < n_tok) {
                v = mi[k];
                if (v >> 16) {
                    len = (int) (v >> 16); d = (int) (v & 0xffff);
                    lc = len_code(len); dc = dist_code(d);
                    nb = S.l_ll[257 + lc] + c_len_extra[lc] + S.l_d[dc] + dist_extra(dc);
                } else {
                    nb = S.l_ll[v];
                }
            }
            int64_t off, sum;
            Scan(scan_tmp).ExclusiveSum((int64_t) nb, off, sum);
            off += carry;
            if (k < n_tok) {
                if (v >> 16) {
                    const int l1 = S.l_ll[257 + lc], e1 = c_len_extra[lc], l2 = S.l_d[dc], e2 = dist_extra(dc);
                    put_bits(words, off, S.c_ll[257 + lc] | ((uint32_t) (len - c_len_base[lc]) << l1), l1 + e1);
                    put_bits(words, off + l1 + e1, S.c_d[dc] | ((uint32_t) (d - c_dist_base[dc]) << l2), l2 + e2);
                } else {
                    put_bits(words, off, S.c_ll[v], S.l_ll[v]);
                }
            }
            __syncthreads();
            if (t == 0) carry += sum;
            __syncthreads();
        }
        if (t == 0) { put_bits(words, carry, S.c_ll[256], S.l_ll[256]); carry += S.l_ll[256]; }
        __syncthreads();
        dbytes = (carry + 7) / 8;
        const uint8_t *wb = reinterpret_cast<const uint8_t *>(words);
        for (int i = t; i < dbytes; i += DF_THREADS) dst[i] = wb[i];
    }
    // gzip member: header with the BC extra field (BSIZE = member bytes - 1), then CRC32 and ISIZE
    const int64_t total = 18 + dbytes + 8;
    if (t == 0) {
        const uint8_t h[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
        for (int k = 0; k < 16; k++) slot[k] = h[k];
        slot[16] = (uint8_t) (total - 1); slot[17] = (uint8_t) ((total - 1) >> 8);
        uint8_t *tr = dst + dbytes;
        const uint32_t crc = S.crc;
        for (int k = 0; k < 4; k++) { tr[k] = (uint8_t) (crc >> (8 * k)); tr[4 + k] = (uint8_t) ((uint32_t) n >> (8 * k)); }
        out_bytes[m] = total;
    }
}

__global__ void k_bgzf_compact(const uint8_t *__restrict__ slots, const int64_t *__restrict__ dst_off, const int64_t *__restrict__ bytes,
                               uint8_t *__restrict__ out) {
    const int m = blockIdx.x;
    const uint8_t *s = slots + (size_t) m * DF_SLOT;
    uint8_t *d = out + dst_off[m];
    const int64_t b = bytes[m];
    for (int64_t i = threadIdx.x; i < b; i += blockDim.x) d[i] = s[i];
}

}  // namespace pb

using namespace pb;

extern "C" int pb_bgzf_compress_device(const uint8_t *d_payload, const int64_t *h_member_off, int64_t n_members, uint8_t *d_out,
                                       int64_t out_cap, int64_t *h_member_bytes, int64_t *n_out, void *stream_) {
    if (!h_member_off || !h_member_bytes || !n_out || n_members < 0) { set_error("null argument"); return PB_ERR_ARG; }
    *n_out = 0;
    for (int64_t k = 0; k < n_members; k++) {
        const int64_t len = h_member_off[k + 1] - h_member_off[k];
        if (len < 0 || len > DF_PAYLOAD) { set_error("member %lld: %lld payload bytes (0..%d)", (long long) k, (long long) len, DF_PAYLOAD); return PB_ERR_ARG; }
    }
    if (n_members == 0) return PB_OK;
    if (!d_payload && h_member_off[n_members] > h_member_off[0]) { set_error("null payload"); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    DevBuf off, scratch, slots, bytes, dst;
    auto run = [&]() -> int {
        PB_CUDA(cudaFuncSetAttribute(k_bgzf_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_SMEM));
        const int64_t batch = n_members < DF_BATCH ? n_members : DF_BATCH;
        PB_TRY(off.reserve(sizeof(int64_t) * (batch + 1))); PB_TRY(dst.reserve(sizeof(int64_t) * batch));
        PB_TRY(bytes.reserve(sizeof(int64_t) * batch));
        PB_TRY(scratch.reserve(sizeof(uint32_t) * DF_PAYLOAD * batch)); PB_TRY(slots.reserve((size_t) DF_SLOT * batch));
        int64_t total = 0;
        std::string err;
        for (int64_t b0 = 0; b0 < n_members; b0 += batch) {
            const int64_t nb = n_members - b0 < batch ? n_members - b0 : batch;
            PB_CUDA(cudaMemcpyAsync(off.p, h_member_off + b0, sizeof(int64_t) * (nb + 1), cudaMemcpyHostToDevice, st));
            k_bgzf_deflate<<<(unsigned) nb, DF_THREADS, DF_SMEM, st>>>(d_payload, off.as<int64_t>(), scratch.as<uint32_t>(),
                                                                     slots.as<uint8_t>(), bytes.as<int64_t>());
            PB_CUDA(cudaGetLastError());
            PB_CUDA(cudaMemcpyAsync(h_member_bytes + b0, bytes.p, sizeof(int64_t) * nb, cudaMemcpyDeviceToHost, st));
            PB_CUDA(cudaStreamSynchronize(st));
            int64_t need = total;
            for (int64_t k = 0; k < nb; k++) need += h_member_bytes[b0 + k];
            if (d_out && need <= out_cap) {
                std::vector<int64_t> h_dst(nb);
                int64_t o = total;
                for (int64_t k = 0; k < nb; k++) { h_dst[k] = o; o += h_member_bytes[b0 + k]; }
                PB_CUDA(cudaMemcpyAsync(dst.p, h_dst.data(), sizeof(int64_t) * nb, cudaMemcpyHostToDevice, st));
                k_bgzf_compact<<<(unsigned) nb, 256, 0, st>>>(slots.as<uint8_t>(), dst.as<int64_t>(), bytes.as<int64_t>(), d_out);
                PB_CUDA(cudaGetLastError());
                PB_CUDA(cudaStreamSynchronize(st));
            }
            total = need;
        }
        *n_out = total;
        if (!d_out || total > out_cap) { set_error("BGZF members need %lld bytes", (long long) total); return PB_ERR_CAPACITY; }
        return PB_OK;
    };
    const int rc = run();
    DevBuf *bufs[] = {&off, &scratch, &slots, &bytes, &dst};
    for (auto *b : bufs) b->release();
    return rc;
}

extern "C" int pb_bgzf_compress_host(const uint8_t *h_payload, const int64_t *h_member_off, int64_t n_members, uint8_t *h_out,
                                     int64_t out_cap, int64_t *h_member_bytes, int64_t *n_out, void *stream_) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) { set_error("no CUDA device: libpepper_b200 has no CPU fallback"); return PB_ERR_CUDA; }
    if (!h_member_off || !h_member_bytes || !n_out || n_members < 0) { set_error("null argument"); return PB_ERR_ARG; }
    *n_out = 0;
    if (n_members == 0) return PB_OK;
    cudaStream_t st = (cudaStream_t) stream_;
    const int64_t lo = h_member_off[0], hi = h_member_off[n_members];
    if (hi < lo) { set_error("member offsets decrease"); return PB_ERR_ARG; }
    DevBuf p, o;
    std::vector<int64_t> rel(n_members + 1);
    for (int64_t k = 0; k <= n_members; k++) rel[k] = h_member_off[k] - lo;
    auto run = [&]() -> int {
        PB_TRY(p.reserve(hi - lo + 1));
        if (hi > lo) PB_TRY(upload(p, h_payload + lo, (size_t) (hi - lo), st));
        PB_TRY(o.reserve(out_cap > 0 ? out_cap : 1));
        const int rc = pb_bgzf_compress_device(p.as<uint8_t>(), rel.data(), n_members, h_out ? o.as<uint8_t>() : nullptr, out_cap,
                                               h_member_bytes, n_out, stream_);
        if (rc != PB_OK) return rc;
        PB_CUDA(cudaMemcpyAsync(h_out, o.p, (size_t) *n_out, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        return PB_OK;
    };
    const int rc = run();
    p.release(); o.release();
    return rc;
}
