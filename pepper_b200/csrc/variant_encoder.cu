// Variant pileup-summary encoder for sm_90a.
//
// Re-design (not a translation) of RegionalSummaryGenerator::generate_summary
// (pepper_variant/modules/cpp/region_summary.cpp:337-916).  The reference walks one read at a
// time and read-modify-writes vector<vector<int>> rows and std::map<string,int> tallies per base.
// Here a batch of regions is processed by six kernels:
//
//   k_cigar_prefix   one warp per read: prefix sums of (reference, read) consumption per CIGAR op
//   k_tile_count     one CTA per 512-position tile: every warp walks the reads overlapping the
//                    tile, counts into shared-memory columns with shared atomics, then the CTA
//                    applies the site thresholds (:634-646) and writes each position's 16 live
//                    matrix columns once (32 B / position)
//   k_site_index     per tile: compacts flagged sites, gives each an event segment
//   k_collect_*      per CIGAR op / per rare base: writes allele events of flagged sites
//   k_site_alleles   one warp per site: dedup + order alleles as std::set<string> would,
//                    apply the candidate filters (:682-712)
//   k_windows        one warp per site: 33x26 int8 window gather + overlay (:828-905), key strings
//
// Only columns 4, 8-15, 19-25 of the 26 are ever non-zero in the base matrix (col 0 is the reference
// code, the rest are written by the per-candidate overlay), so 16 int16 are stored per position.
#include "handles.cuh"
#include <vector>
#include <algorithm>

namespace pb {

constexpr int TILE = 512;            // positions per k_tile_count CTA
constexpr int TC_THREADS = 256;
constexpr int LIST_CAP = 1024;       // reads scanned per round of k_tile_count
constexpr int MAX_KEY = 61;          // region_summary.cpp:461,511 candidate_string.length() <= 61

// shared-memory counter columns of k_tile_count (int32 [NCNT][TILE])
enum {
    C_TOT_F = 0, C_TOT_R,          // M bases with q >= min_snp_baseq per strand
    C_ANC_F, C_ANC_R,              // ... of which anchor an I/D (excluded from REFF/REFR, :381-391)
    C_A_F, C_C_F, C_G_F, C_T_F,    // bases whose column differs from the reference column
    C_A_R, C_C_R, C_G_R, C_T_R,
    C_NON_F, C_NON_R,              // non-ACGT read bases
    C_I_F, C_I_R,                  // col 12 / 23
    C_D_F, C_D_R,                  // col 13 / 24 (deletion anchors + IUPAC 'D' bases)
    C_S_F, C_S_R,                  // col 14 / 25 ('*' + other bases)
    C_COVX,                        // coverage increments of :453
    C_SNP, C_INS, C_DEL,           // snp_count / insert_count / delete_count
    C_RARE,                        // SNP alleles that cannot be derived from the columns
    NCNT
};

// per-position meta word: bit0 snp pass, bit1 insert pass, bit2 delete pass, bit3 site; bits 4.. event slots
constexpr uint32_t F_SNP = 1, F_INS = 2, F_DEL = 4, F_SITE = 8;

struct RareEv { uint32_t g; uint8_t code; uint8_t strand; uint16_t pad; };

struct Ev {            // 40 B allele event / allele entry
    uint64_t key;      // order key inside a type (see ins_key / klen / ascii rank)
    uint32_t read;     // source read (insert bases)
    uint32_t ridx;     // index of the anchor base in the read
    uint16_t klen;     // bases in the key after the type digit
    uint8_t type;      // 1 snp, 2 insert, 3 delete
    uint8_t strand;
    uint8_t leader;
    uint8_t pass;
    uint8_t code;      // snp: NT16 code
    uint8_t pad;
    int32_t total, fwd;
    int32_t order;
    int32_t pad2;
};

struct Cand {          // 32 B candidate record
    uint32_t read, ridx;
    int32_t total, fwd, rev;
    uint16_t klen;
    uint8_t type, code;
    uint32_t pad[2];
};

struct DevReads {
    const int64_t *pos, *seq_off, *cigar_off;
    const uint8_t *flags, *mapq, *seq, *qual;
    const uint32_t *cigar;
    int64_t n_reads;
};

struct VParams {
    int minq_snp;                 // ceil(min_snp_baseq): integer q >= min_snp_baseq  <=>  q >= ceil
    double min_snp_baseq, min_indel_baseq;
    double snp_thr, ins_thr, del_thr, min_cov, snp_cand_thr, indel_cand_thr, support_thr;
    int skip_indels;
};

// ------------------------------------------------------------------ k_cigar_prefix
// Consumption rules of the walker (region_summary.cpp:356-563): M/=/X ref+read; I read; D ref;
// N and P advance ref AND (falling through into S, :556-560) read; S read; H nothing.
__device__ __forceinline__ void op_consumes(uint32_t w, int &dref, int &drd) {
    const int op = w & 15, len = (int) (w >> 4);
    dref = 0; drd = 0;
    switch (op) {
        case 0: case 7: case 8: dref = len; drd = len; break;
        case 1: drd = len; break;
        case 2: dref = len; break;
        case 3: case 6: dref = len; drd = len; break;
        case 4: drd = len; break;
        default: break;
    }
}

// One warp per read; every lane takes 4 consecutive ops of a 128-op chunk (lane-local prefix, one warp scan of the lane sums),
// and the next chunk's words are in flight while this one is scanned: the longest read of a batch bounds the launch, so the
// serial chunk count per read is what matters.
__global__ void k_cigar_prefix(DevReads R, int32_t *__restrict__ op_ref, int32_t *__restrict__ op_rd,
                               int32_t *__restrict__ read_reflen) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= R.n_reads) return;
    const int64_t c0 = R.cigar_off[r], c1 = R.cigar_off[r + 1];
    int cref = 0, crd = 0;
    uint32_t nx[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { const int64_t i = c0 + 4 * lane + k; nx[k] = (i < c1) ? __ldg(R.cigar + i) : 5u; }   // 5 = H: consumes nothing
    for (int64_t c = c0; c < c1; c += 128) {
        const int64_t b = c + 4 * lane;
        uint32_t w[4];
#pragma unroll
        for (int k = 0; k < 4; k++) { w[k] = nx[k]; const int64_t i = b + 128 + k; nx[k] = (i < c1) ? __ldg(R.cigar + i) : 5u; }
        int dr[4], dd[4], lref = 0, lrd = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) { op_consumes(w[k], dr[k], dd[k]); lref += dr[k]; lrd += dd[k]; }
        int sref = lref, srd = lrd;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            int a = __shfl_up_sync(0xffffffffu, sref, d), bb = __shfl_up_sync(0xffffffffu, srd, d);
            if (lane >= d) { sref += a; srd += bb; }
        }
        int pref = cref + sref - lref, prd = crd + srd - lrd;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (b + k < c1) { op_ref[b + k] = pref; op_rd[b + k] = prd; }
            pref += dr[k]; prd += dd[k];
        }
        cref += __shfl_sync(0xffffffffu, sref, 31);
        crd += __shfl_sync(0xffffffffu, srd, 31);
    }
    if (lane == 0) read_reflen[r] = cref;
}

// ------------------------------------------------------------------ shared op predicates
// Insert allele of one I op (region_summary.cpp:431-488).  Returns true when the allele is tallied;
// cov_extra is the coverage increment of :453.
__device__ __forceinline__ bool insert_allele(const DevReads &R, int64_t so, int64_t lseq, int rd_idx, int len,
                                              const VParams &P, int &klen, bool &cov_extra) {
    const int64_t s = (int64_t) rd_idx - 1;
    const int64_t n = (int64_t) len + 1;
    // (sum of small integers: exact in the reference's double accumulator, so an integer sum compares identically; four
    //  independent loads per step instead of one dependent add per load)
    const uint8_t *qp = R.qual + so + s;
    long long qs = 0;
    int64_t i = 0;
    for (; i + 4 <= n; i += 4) {
        const int q0 = __ldg(qp + i), q1 = __ldg(qp + i + 1), q2 = __ldg(qp + i + 2), q3 = __ldg(qp + i + 3);
        qs += (q0 + q1) + (q2 + q3);
    }
    for (; i < n; i++) qs += __ldg(qp + i);
    const bool qok = (double) qs >= P.min_indel_baseq * (double) n;
    cov_extra = qok && ((double) __ldg(R.qual + so + s) < P.min_snp_baseq);
    int64_t k = n;
    if (s + k > lseq) k = lseq - s;          // std::string::substr clamps
    klen = (int) k;
    return (1 + k <= MAX_KEY) && qok;
}
// Delete allele key length (region_summary.cpp:500,507-511): "3" + reference.substr(x, len+1)
__device__ __forceinline__ bool delete_allele(int64_t x, int len, int64_t ref_len, int &klen) {
    int64_t k = (int64_t) len + 1;
    if (x + k > ref_len) k = ref_len - x;
    if (k < 0) k = 0;
    klen = (int) k;
    return 1 + k <= MAX_KEY;
}

// class of a read base: 0..3 = A,C,G,T  4 = IUPAC 'D' (lands in the D column, region_summary.cpp:214)  5 = other
__device__ __forceinline__ int base_class(int code) {
    // code: 0 1 2 3 4 5 6 7 8 9 10 11 12 13 14 15
    //       5 0 1 5 2 5 5 5 3 5  5  5  5  4  5  5
    return (int) ((0x5545555355525105ULL >> (4 * code)) & 15ULL);
}
// class of a reference character: 0..3 valid (case-insensitive, check_ref_base :193), 7 invalid
__device__ __forceinline__ int ref_class(char c) {
    switch (to_upper(c)) { case 'A': return 0; case 'C': return 1; case 'G': return 2; case 'T': return 3; default: return 7; }
}

// ------------------------------------------------------------------ k_tile_count
struct TileArgs {
    DevReads R;
    const pb_region_t *regions;
    const char *ref;
    const int32_t *op_ref, *op_rd, *read_reflen;
    const int32_t *tile_region;      // [n_tiles]
    const int32_t *tile_x0;          // [n_tiles] first position of the tile relative to ref_start
    const int64_t *region_goff;      // [n_regions] global position index of the region's first position
    int16_t *M16;                    // [G][16]
    int32_t *cov;                    // [G]
    uint32_t *meta;                  // [G]
    int32_t *dbg_counts;             // optional [G][3] snp, ins, del
    int32_t *tile_nsites, *tile_nev; // [n_tiles]
    RareEv *rare; unsigned long long *rare_n; unsigned long long rare_cap;
    uint32_t *track;                 // optional gVCF track: (n_ref | n_alt << 16) per owned position
    const int64_t *track_reg;        // [n_regions][2] track offset of cand_start, owned end (absolute, inclusive)
    VParams P;
};

__global__ void __launch_bounds__(TC_THREADS, 4) k_tile_count(TileArgs A) {
    extern __shared__ int32_t smem[];
    int32_t *cnt = smem;                                   // [NCNT][TILE]
    char *s_ref = reinterpret_cast<char *>(cnt + NCNT * TILE);   // [TILE]
    uint8_t *s_rinfo = reinterpret_cast<uint8_t *>(s_ref + TILE);  // [TILE]
    __shared__ int s_red[2];
    __shared__ int s_list[LIST_CAP];
    __shared__ int s_nlist, s_next;

    const int t = blockIdx.x;
    const int reg = A.tile_region[t];
    const pb_region_t rg = A.regions[reg];
    const int64_t x0 = A.tile_x0[t];
    const int64_t L1 = rg.ref_end - rg.ref_start + 1;
    const int npos = (int) min((int64_t) TILE, L1 - x0);
    const int64_t lo = rg.ref_start + x0, hi = lo + npos - 1;      // absolute, inclusive
    const int tid = threadIdx.x, lane = tid & 31;

    for (int i = tid; i < NCNT * TILE; i += TC_THREADS) cnt[i] = 0;
    for (int i = tid; i < TILE; i += TC_THREADS) {
        const int64_t x = x0 + i;
        const char c = (i < npos && x < rg.ref_len) ? A.ref[rg.ref_off + x] : '\0';
        s_ref[i] = c;
        // bits 0-3: NT16 code of the reference character, bit 4: not an (upper-case) NT16 character -> every read base
        // mismatches it (raw char compare, region_summary.cpp:394), bits 5-7: column class (0-3 = A,C,G,T; 7 = invalid)
        int code = 16;
#pragma unroll
        for (int k = 0; k < 16; k++) if (c == nt16_char(k)) code = k;
        s_rinfo[i] = (uint8_t) (code | (ref_class(c) << 5));
    }
    if (tid < 2) s_red[tid] = 0;
    if (tid == 0) { s_nlist = 0; s_next = 0; }
    __syncthreads();

    const DevReads &R = A.R;
    const VParams &P = A.P;
    const bool minq_all = P.minq_snp > 255;                          // no 8-bit quality can pass
    const uint32_t minq4 = (uint32_t) max(0, min(P.minq_snp, 255)) * 0x01010101u;

    // ---- overlapping reads are first compacted into a shared list (reads are position sorted, so the ones touching a
    //      tile are neighbours: handing out groups of 32 consecutive reads per warp would leave most warps idle),
    //      then warps take reads from the list dynamically
    for (int64_t blk = rg.read_begin; blk < rg.read_end; blk += LIST_CAP) {
        const int64_t blk_end = min(rg.read_end, blk + (int64_t) LIST_CAP);
        for (int64_t rmine = blk + tid; rmine < blk_end; rmine += TC_THREADS) {
            if (__ldg(R.mapq + rmine) > 0 && R.seq_off[rmine + 1] > R.seq_off[rmine]) {
                const int64_t p0 = __ldg(R.pos + rmine);
                const int64_t p1 = p0 + __ldg(A.read_reflen + rmine);      // exclusive end
                // ops of interest touch [lo-1 .. hi+1]
                if ((p0 <= hi + 1) && (p1 >= lo - 1)) s_list[atomicAdd(&s_nlist, 1)] = (int) (rmine - blk);
            }
        }
        __syncthreads();
        const int nlist = s_nlist;
        while (true) {
            int item = 0;
            if (lane == 0) item = atomicAdd(&s_next, 1);
            item = __shfl_sync(0xffffffffu, item, 0);
            if (item >= nlist) break;
            const int64_t r = blk + s_list[item];
            {
            const int64_t rpos = __ldg(R.pos + r);
            const int64_t so = R.seq_off[r];
            const int64_t lseq = R.seq_off[r + 1] - so;
            const int64_t c0 = R.cigar_off[r], c1 = R.cigar_off[r + 1];
            const int nops = (int) (c1 - c0);
            const int rev = __ldg(R.flags + r) & 1;
            // --- first op to look at: last op whose start <= lo - rpos (32-ary cooperative search)
            const int64_t target = lo - rpos;
            int first = 0;
            if (target > 0) {
                int base = 0, n = nops;
                while (n > 1) {
                    const int stride = (n + 31) / 32;
                    const int idx = base + lane * stride;
                    const bool le = (lane * stride < n) && ((int64_t) __ldg(A.op_ref + c0 + idx) <= target);
                    const unsigned m = __ballot_sync(0xffffffffu, le);
                    const int k = __popc(m);                 // op_ref is non-decreasing: a prefix of lanes
                    if (k == 0) { n = 0; break; }
                    const int nb = base + (k - 1) * stride;
                    n = min(stride, base + n - nb);
                    base = nb;
                }
                first = base;
            }
            // --- walk chunks of 32 ops (all positions below are int32, relative to the tile start `lo`)
            const int rpos_rel = (int) (rpos - lo);
            const int end_rel = (int) (rg.ref_end - lo);
            const int hi_rel = npos - 1;
            for (int j0 = first; j0 < nops; j0 += 32) {
                const int j = j0 + lane;
                uint32_t w = 0; int pr = 0, pd = 0;
                if (j < nops) { w = __ldg(R.cigar + c0 + j); pr = __ldg(A.op_ref + c0 + j); pd = __ldg(A.op_rd + c0 + j); }
                uint32_t wn = __shfl_down_sync(0xffffffffu, w, 1);
                if (lane == 31) wn = (j + 1 < nops) ? __ldg(R.cigar + c0 + j + 1) : 0xfu;
                if (j + 1 >= nops) wn = 0xfu;                   // no next op
                const int op = (j < nops) ? (int) (w & 15) : 15;
                const int len = (int) (w >> 4);
                const int a = rpos_rel + pr;                    // ref position at op start, relative to lo
                const bool live = (j < nops) && (a <= end_rel);        // walker breaks when ref_position > ref_end (:355)
                // chunk exit test: every later op starts at or after this chunk's last start
                const int a_last = __shfl_sync(0xffffffffu, a, 31);
                const bool is_m = (op == 0 || op == 7 || op == 8);
                // clipped per-position segment (M bases or deleted positions)
                int s0 = 0, scnt = 0;
                if (live && (is_m || op == 2)) {
                    const int b0 = max(a, 0), b1 = min(a + len - 1, hi_rel);
                    if (b1 >= b0) { s0 = b0; scnt = b1 - b0 + 1; }
                }
                // anchor of an I/D after the last base of this M op
                const int nop = (int) (wn & 15);
                const int op_last = (is_m && (nop == 1 || nop == 2)) ? a + len - 1 : -0x40000000;
                // --- I / D ops anchored in this tile (handled by the op's own lane)
                if (live && (op == 1 || op == 2)) {
                    const int x = a - 1;
                    if (x >= 0 && x <= hi_rel) {
                        const bool rvalid = ref_class(s_ref[x]) < 4;
                        if (op == 1) {
                            if (pd >= 1) {
                                int klen; bool covx;
                                const bool ok = insert_allele(R, so, lseq, pd, len, P, klen, covx);
                                if (covx) atomicAdd(&cnt[C_COVX * TILE + x], 1);
                                if (ok) {
                                    if (rvalid) atomicAdd(&cnt[(C_I_F + rev) * TILE + x], 1);
                                    atomicAdd(&cnt[C_INS * TILE + x], 1);
                                }
                            }
                        } else {
                            if (rvalid) atomicAdd(&cnt[(C_D_F + rev) * TILE + x], 1);
                            int klen;
                            if (delete_allele(x0 + x, len, rg.ref_len, klen)) atomicAdd(&cnt[C_DEL * TILE + x], 1);
                        }
                    }
                }
                // --- range counters as difference arrays (prefix-summed in the epilogue): every M op adds its clipped segment to
                //     the strand's base total, every D op to the strand's '*' column — two atomics per op instead of one per base
                if (scnt > 0) {
                    int32_t *d = cnt + ((is_m ? C_TOT_F : C_S_F) + rev) * TILE;
                    atomicAdd(d + s0, 1);
                    if (s0 + scnt <= hi_rel) atomicAdd(d + s0 + scnt, -1);
                }
                // --- per-base work of the M ops, balanced over the warp in QUADS of 4 consecutive bases of one op: a quad whose
                //     bases all pass the quality threshold and equal the reference character needs nothing beyond the range add
                const int nq = is_m ? (scnt + 3) >> 2 : 0;
                int incl = nq;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int v = __shfl_up_sync(0xffffffffu, incl, d);
                    if (lane >= d) incl += v;
                }
                const int total = __shfl_sync(0xffffffffu, incl, 31);
                const int excl = incl - nq;
                const int base_x = s0 - 4 * excl;                           // x of the first base of quad idx: base_x + 4 idx
                const int base_rd = pd + (s0 - a) - 4 * excl;               // read index of that base
                // exclusive end of the segment, bit 0: the segment's last base anchors an I/D (and lies in this tile)
                const int pk = ((s0 + scnt) << 1) | ((nq > 0 && op_last == s0 + scnt - 1) ? 1 : 0);
                for (int k0 = 0; k0 < total; k0 += 32) {
                    const int idx = k0 + lane;
                    // smallest l with incl[l] > idx
                    int l = 0;
#pragma unroll
                    for (int step = 16; step >= 1; step >>= 1) {
                        const int v = __shfl_sync(0xffffffffu, incl, l + step - 1);
                        if (v <= idx) l += step;
                    }
                    l = min(l, 31);
                    const int o_bx = __shfl_sync(0xffffffffu, base_x, l);
                    const int o_brd = __shfl_sync(0xffffffffu, base_rd, l);
                    const int o_pk = __shfl_sync(0xffffffffu, pk, l);
                    if (idx < total) {
                        const int xq = o_bx + 4 * idx;
                        const int nb = min(4, (o_pk >> 1) - xq);            // bases of this quad (1..4)
                        const int64_t ri = so + (int64_t) (o_brd + 4 * idx);
                        const uint8_t *qp = R.qual + ri;
                        const uint8_t *sp = R.seq + (ri >> 1);
                        const int odd = (int) (ri & 1);
                        // qualities / reference info of the quad, one byte per base; the 4-bit codes as a 24-bit nibble stream
                        uint32_t qw = __ldg(qp), rw = s_rinfo[xq], sw = (uint32_t) __ldg(sp) << 16;
                        if (nb > 1) { qw |= (uint32_t) __ldg(qp + 1) << 8; rw |= (uint32_t) s_rinfo[xq + 1] << 8; }
                        if (nb > 2) { qw |= (uint32_t) __ldg(qp + 2) << 16; rw |= (uint32_t) s_rinfo[xq + 2] << 16; }
                        if (nb > 3) { qw |= (uint32_t) __ldg(qp + 3) << 24; rw |= (uint32_t) s_rinfo[xq + 3] << 24; }
                        if (odd + nb > 2) sw |= (uint32_t) __ldg(sp + 1) << 8;
                        if (odd + nb > 4) sw |= (uint32_t) __ldg(sp + 2);
                        sw >>= 4 * (1 - odd);                               // base k of the quad: bits [19 - 4k, 16 - 4k]
                        // codes spread to one byte per base (byte k = base k), then byte-wise SIMD tests of the whole quad
                        uint32_t cw = (sw >> 4) & 0xffffu;
                        cw = (cw | (cw << 8)) & 0x00ff00ffu;
                        cw = (cw | (cw << 4)) & 0x0f0f0f0fu;
                        cw = __byte_perm(cw, 0, 0x0123);
                        unsigned ex = (__vcmpne4(cw, rw & 0x1f1f1f1fu) | (minq_all ? 0xffffffffu : __vcmpltu4(qw, minq4))) &
                                      (0xffffffffu >> (8 * (4 - nb)));
                        if (o_pk & 1) {                                     // anchor of an I/D: the last base of the segment (:381-391)
                            const int ka = (o_pk >> 1) - 1 - xq;
                            if (ka < nb && (int) ((qw >> (8 * ka)) & 255u) >= P.minq_snp)
                                atomicAdd(&cnt[(C_ANC_F + rev) * TILE + xq + ka], 1);
                        }
                        while (ex) {
                            const int k = (__ffs((int) ex) - 1) >> 3;
                            ex &= ~(0xffu << (8 * k));
                            const int x = xq + k;
                            const int q = (int) ((qw >> (8 * k)) & 255u);
                            if (q < P.minq_snp) {                           // not a counted base: take it out of the range total
                                atomicAdd(&cnt[(C_TOT_F + rev) * TILE + x], -1);
                                if (x < hi_rel) atomicAdd(&cnt[(C_TOT_F + rev) * TILE + x + 1], 1);
                                continue;
                            }
                            const int code = (int) ((cw >> (8 * k)) & 15u);
                            const uint32_t rinfo = (rw >> (8 * k)) & 255u;
                            const int rcls = (int) (rinfo >> 5);
                            const int cls = base_class(code);
                            // column differing from the reference column
                            if (rcls < 4 && cls != rcls) {
                                if (cls < 4) {
                                    atomicAdd(&cnt[(C_A_F + 4 * rev + cls) * TILE + x], 1);
                                } else {
                                    atomicAdd(&cnt[(C_NON_F + rev) * TILE + x], 1);
                                    if (cls == 4) atomicAdd(&cnt[(C_D_F + rev) * TILE + x], 1);
                                    else {                                  // point add to the '*' difference array
                                        atomicAdd(&cnt[(C_S_F + rev) * TILE + x], 1);
                                        if (x < hi_rel) atomicAdd(&cnt[(C_S_F + rev) * TILE + x + 1], -1);
                                    }
                                }
                            }
                            // nt16_char(code) != reference character (always true here: the quad test let equal bases through)
                            atomicAdd(&cnt[C_SNP * TILE + x], 1);
                            if (rcls >= 4 || cls >= 4) {
                                atomicAdd(&cnt[C_RARE * TILE + x], 1);
                                const unsigned long long slot = atomicAdd(A.rare_n, 1ULL);
                                if (slot < A.rare_cap) {
                                    RareEv e; e.g = (uint32_t) (A.region_goff[reg] + x0 + x); e.code = (uint8_t) code;
                                    e.strand = (uint8_t) rev; e.pad = 0;
                                    A.rare[slot] = e;
                                }
                            }
                        }
                    }
                }
                if (a_last > hi_rel + 1) break;  // warp-uniform: later ops cannot touch the tile
            }
            }
        }
        __syncthreads();
        if (tid == 0) { s_nlist = 0; s_next = 0; }
        __syncthreads();
    }

    // ---- the four difference arrays (base totals and '*' columns per strand) -> counts: block-wide inclusive prefix sums,
    //      two positions per thread
    {
        __shared__ int s_wsum[4][TC_THREADS / 32];
        static_assert(TILE == 2 * TC_THREADS, "the scan below takes two positions per thread");
        const int cols[4] = {C_TOT_F, C_TOT_R, C_S_F, C_S_R};
        int v0[4], v1[4], inc[4];
#pragma unroll
        for (int c = 0; c < 4; c++) {
            v0[c] = cnt[cols[c] * TILE + 2 * tid];
            v1[c] = cnt[cols[c] * TILE + 2 * tid + 1];
            inc[c] = v0[c] + v1[c];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, inc[c], d);
                if (lane >= d) inc[c] += v;
            }
            if (lane == 31) s_wsum[c][tid >> 5] = inc[c];
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < 4; c++) {
            int off = 0;
            for (int w = 0; w < (tid >> 5); w++) off += s_wsum[c][w];
            const int before = off + inc[c] - v0[c] - v1[c];
            cnt[cols[c] * TILE + 2 * tid] = before + v0[c];
            cnt[cols[c] * TILE + 2 * tid + 1] = before + v0[c] + v1[c];
        }
        __syncthreads();
    }

    // ---- epilogue: derive the columns, site thresholds (region_summary.cpp:634-646), one write per position
    const int64_t g0 = A.region_goff[reg] + x0;
    int my_sites = 0, my_ev = 0;
    for (int x = tid; x < npos; x += TC_THREADS) {
#define CN(c) cnt[(c) * TILE + x]
        const int rcls = ref_class(s_ref[x]);
        const int cov = CN(C_TOT_F) + CN(C_TOT_R) + CN(C_COVX);
        int16_t row[16];
        row[0] = (int16_t) -(CN(C_TOT_F) - CN(C_ANC_F));           // col 4  REFF
        row[8] = (int16_t) -(CN(C_TOT_R) - CN(C_ANC_R));           // col 15 REFR
#pragma unroll
        for (int s = 0; s < 2; s++) {
            int n[4];
            int others = CN(C_NON_F + s);
#pragma unroll
            for (int b = 0; b < 4; b++) { n[b] = CN(C_A_F + 4 * s + b); others += n[b]; }
            if (rcls < 4) {
#pragma unroll
                for (int b = 0; b < 4; b++) if (b == rcls) n[b] = CN(C_TOT_F + s) - others;
            }
            const int o = s ? 9 : 1;                                   // cols 19.. / 8..
#pragma unroll
            for (int b = 0; b < 4; b++) row[o + b] = (int16_t) -((rcls < 4) ? n[b] : 0);
            row[o + 4] = (int16_t) -CN(C_I_F + s);
            row[o + 5] = (int16_t) -CN(C_D_F + s);
            row[o + 6] = (int16_t) -((rcls < 4) ? CN(C_S_F + s) : 0);     // deleted positions count only over a valid reference base
        }
        const int64_t g = g0 + x;
        int4 *dst = reinterpret_cast<int4 *>(A.M16 + g * 16);
        const int4 *srcv = reinterpret_cast<const int4 *>(row);
        dst[0] = srcv[0];
        dst[1] = srcv[1];
        A.cov[g] = cov;
        // gVCF track: reference / non-reference counts of an owned position over both strands, from the unclamped columns
        // (n_ref = count(R) - I - D, n_alt = the other bases + '*' + I + D; zero over a non-ACGT reference)
        if (A.track) {
            const int64_t pos = lo + x, t0 = A.track_reg[2 * reg], own_end = A.track_reg[2 * reg + 1];
            if (pos >= rg.cand_start && pos <= own_end) {
                uint32_t v = 0;
                if (rcls < 4) {
                    const int ins = -((int) row[5] + row[13]), del = -((int) row[6] + row[14]), oth = -((int) row[7] + row[15]);
                    int nalt = ins + del + oth, nref = 0;
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        const int c = -((int) row[1 + b] + row[9 + b]);
                        if (b == rcls) nref = c; else nalt += c;
                    }
                    nref = max(0, nref - ins - del);
                    v = (uint32_t) min(nref, 65535) | ((uint32_t) min(max(nalt, 0), 65535) << 16);
                }
                A.track[t0 + pos - rg.cand_start] = v;
            }
        }
        const int snp = CN(C_SNP), ins = CN(C_INS), del = CN(C_DEL);
        if (A.dbg_counts) { A.dbg_counts[g * 3] = snp; A.dbg_counts[g * 3 + 1] = ins; A.dbg_counts[g * 3 + 2] = del; }
        const double c = fmax(1.0, (double) cov);
        const double fs = (double) snp / c, fi = (double) ins / c, fd = (double) del / c;
        uint32_t m = 0;
        const int64_t pos = lo + x;
        if ((fs >= P.snp_thr || fi >= P.ins_thr || fd >= P.del_thr) && pos >= rg.cand_start && pos <= rg.cand_end &&
            (double) cov >= P.min_cov) {
            m = F_SITE;
            int ev = 0;
            if (fs >= P.snp_thr) { m |= F_SNP; ev += 4 + CN(C_RARE); }
            if (fi >= P.ins_thr) { m |= F_INS; ev += ins; }
            if (fd >= P.del_thr) { m |= F_DEL; ev += del; }
            m |= (uint32_t) ev << 4;
            my_sites += 1;
            my_ev += ev;
        }
        A.meta[g] = m;
#undef CN
    }
    atomicAdd(&s_red[0], my_sites);
    atomicAdd(&s_red[1], my_ev);
    __syncthreads();
    if (tid == 0) { A.tile_nsites[t] = s_red[0]; A.tile_nev[t] = s_red[1]; }
}

// ------------------------------------------------------------------ k_site_index
struct SiteArgs {
    const pb_region_t *regions;
    const int32_t *tile_region, *tile_x0;
    const int64_t *region_goff;
    const uint32_t *meta;
    const int64_t *tile_site_base, *tile_ev_base;
    uint32_t *site_of;       // [G] (valid where flagged)
    uint32_t *site_g;        // [n_sites]
    int64_t *site_evoff;     // [n_sites+1]
    int64_t n_sites_total, n_ev_total;
};

__global__ void __launch_bounds__(TILE) k_site_index(SiteArgs A) {
    __shared__ int s_ws[TILE / 32], s_we[TILE / 32];
    const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int reg = A.tile_region[t];
    const pb_region_t rg = A.regions[reg];
    const int64_t x0 = A.tile_x0[t];
    const int64_t L1 = rg.ref_end - rg.ref_start + 1;
    const int npos = (int) min((int64_t) TILE, L1 - x0);
    const int64_t g = A.region_goff[reg] + x0 + tid;
    uint32_t m = (tid < npos) ? A.meta[g] : 0;
    int fs = (m & F_SITE) ? 1 : 0, fe = (int) (m >> 4);
    int is = fs, ie = fe;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, is, d), b = __shfl_up_sync(0xffffffffu, ie, d);
        if (lane >= d) { is += a; ie += b; }
    }
    if (lane == 31) { s_ws[warp] = is; s_we[warp] = ie; }
    __syncthreads();
    int bs = 0, be = 0;
    for (int w = 0; w < warp; w++) { bs += s_ws[w]; be += s_we[w]; }
    if (fs) {
        const int64_t s = A.tile_site_base[t] + bs + is - 1;
        A.site_of[g] = (uint32_t) s;
        A.site_g[s] = (uint32_t) g;
        A.site_evoff[s] = A.tile_ev_base[t] + be + ie - fe;
    }
    if (t == 0 && tid == 0) A.site_evoff[A.n_sites_total] = A.n_ev_total;
}

// ------------------------------------------------------------------ k_collect_ops / k_collect_rare
// 5 bits per base (ascii rank + 1), first 12 bases, most significant first: numeric order == std::string order
__device__ __forceinline__ uint64_t ins_key(const DevReads &R, int64_t so, int64_t s, int klen) {
    uint64_t k = 0;
    const int n = min(klen, 12);
    for (int i = 0; i < n; i++) {
        const uint64_t sym = (uint64_t) nt16_ascii_rank(seq_code_at(R.seq, so + s + i)) + 1ULL;
        k |= sym << (5 * (11 - i));
    }
    return k;
}

struct CollectArgs {
    DevReads R;
    const pb_region_t *regions;
    const int32_t *read_region;
    const int64_t *region_goff;
    const int32_t *op_ref, *op_rd;
    const uint32_t *meta, *site_of;
    const int64_t *site_evoff;
    uint32_t *site_cur;
    Ev *ev;
    const RareEv *rare; unsigned long long n_rare;
    int64_t op_first, op_last;       // the batch's op range in R.cigar / op_ref / op_rd
    VParams P;
};

__device__ __forceinline__ Ev *claim_slot(const CollectArgs &A, uint32_t m, uint32_t s) {
    const uint32_t k = atomicAdd(A.site_cur + s, 1u);
    return A.ev + A.site_evoff[s] + ((m & F_SNP) ? 4 : 0) + k;
}

// Flat over the batch's CIGAR ops: a warp takes COLLECT_CHUNK consecutive ops of the op array, whichever reads they belong to
// (one warp per read made the longest read of a batch — 20 k ops of a 100 kb ONT read — the duration of the launch).  The read
// of the chunk's first op comes from one cooperative search in cigar_off; after that every lane walks its own read index forward.
constexpr int COLLECT_CHUNK = 1024;

__global__ void k_collect_ops(CollectArgs A) {
    const int lane = threadIdx.x & 31;
    const int64_t wid = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const DevReads &R = A.R;
    const int64_t c_beg = A.op_first + wid * COLLECT_CHUNK;
    if (c_beg >= A.op_last) return;
    const int64_t c_end = min(A.op_last, c_beg + (int64_t) COLLECT_CHUNK);
    // largest r with cigar_off[r] <= c_beg (32-ary: cigar_off is non-decreasing, so the lanes that pass form a prefix)
    int64_t r = 0;
    {
        int64_t base = 0, n = R.n_reads;
        while (n > 1) {
            const int64_t stride = (n + 31) / 32;
            const int64_t off = (int64_t) lane * stride;
            const bool le = (off < n) && (R.cigar_off[base + off] <= c_beg);
            const int k = __popc(__ballot_sync(0xffffffffu, le));
            if (k == 0) { n = 0; break; }
            const int64_t nb = base + (int64_t) (k - 1) * stride;
            n = min(stride, base + n - nb);
            base = nb;
        }
        r = base;
    }
    int64_t r_have = -1;
    bool skip = true;
    int64_t so = 0, lseq = 0, rpos = 0, goff = 0, ref_start = 0, ref_end = 0, ref_len = 0, next_off = R.cigar_off[r + 1];
    int rev = 0;
    for (int64_t c4 = c_beg + lane; c4 < c_end; c4 += 128) {
        uint32_t w4[4]; int pr4[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int64_t c = c4 + 32 * k;
            const bool in = c < c_end;
            w4[k] = in ? __ldg(R.cigar + c) : 0u;
            pr4[k] = in ? __ldg(A.op_ref + c) : 0;
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int64_t c = c4 + 32 * k;
            const uint32_t w = w4[k];
            const int op = w & 15, len = (int) (w >> 4);
            if (op != 1 && op != 2) continue;
            while (c >= next_off) { r++; next_off = R.cigar_off[r + 1]; }
            if (r != r_have) {
                r_have = r;
                so = R.seq_off[r]; lseq = R.seq_off[r + 1] - so;
                const int reg = A.read_region[r];
                skip = (R.mapq[r] == 0) || (lseq == 0) || (reg < 0);
                if (!skip) {
                    const pb_region_t *rg = A.regions + reg;
                    ref_start = rg->ref_start; ref_end = rg->ref_end; ref_len = rg->ref_len;
                    goff = A.region_goff[reg];
                    rpos = R.pos[r];
                    rev = R.flags[r] & 1;
                }
            }
            if (skip) continue;
            const int64_t a = rpos + pr4[k];
            if (a > ref_end) continue;                          // :355
            const int64_t p = a - 1;
            if (p < ref_start || p > ref_end) continue;
            const int64_t x = p - ref_start;
            const int64_t g = goff + x;
            const uint32_t m = A.meta[g];
            if (op == 1) {
                if (!(m & F_INS)) continue;
                const int pd = __ldg(A.op_rd + c);
                if (pd < 1) continue;
                int klen; bool covx;
                if (!insert_allele(R, so, lseq, pd, len, A.P, klen, covx)) continue;
                Ev *e = claim_slot(A, m, A.site_of[g]);
                Ev v; memset(&v, 0, sizeof(v));
                v.type = 2; v.strand = (uint8_t) rev; v.klen = (uint16_t) klen; v.read = (uint32_t) r; v.ridx = (uint32_t) (pd - 1);
                v.key = ins_key(R, so, pd - 1, klen);
                *e = v;
            } else {
                if (!(m & F_DEL)) continue;
                int klen;
                if (!delete_allele(x, len, ref_len, klen)) continue;
                Ev *e = claim_slot(A, m, A.site_of[g]);
                Ev v; memset(&v, 0, sizeof(v));
                v.type = 3; v.strand = (uint8_t) rev; v.klen = (uint16_t) klen; v.key = (uint64_t) klen;
                *e = v;
            }
        }
    }
}

__global__ void k_collect_rare(CollectArgs A) {
    const unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n_rare) return;
    const RareEv re = A.rare[i];
    const uint32_t m = A.meta[re.g];
    if (!(m & F_SNP)) return;
    Ev *e = claim_slot(A, m, A.site_of[re.g]);
    Ev v; memset(&v, 0, sizeof(v));
    v.type = 1; v.strand = re.strand; v.klen = 1; v.code = re.code; v.key = (uint64_t) nt16_ascii_rank(re.code);
    *e = v;
}

// ------------------------------------------------------------------ k_site_alleles
struct AlleleArgs {
    DevReads R;
    const pb_region_t *regions;
    const char *ref;
    const int64_t *region_goff;      // [n_regions+1]
    int64_t n_regions;
    const uint32_t *site_g;
    const int64_t *site_evoff;
    const int16_t *M16;
    const int32_t *cov;
    const uint32_t *meta;
    Ev *ev;
    Cand *cand_tmp;                  // same indexing as ev
    int32_t *site_ncand;
    int32_t *site_region;            // [n_sites] (written here, reused by k_windows)
    int64_t n_sites;
    VParams P;
};

__device__ __forceinline__ int find_region(const int64_t *goff, int64_t n_regions, int64_t g) {
    int lo = 0, hi = (int) n_regions - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (goff[mid] <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// tails (bases 12..) of two insert alleles: <0, 0, >0 like std::string::compare
__device__ int ins_tail_cmp(const DevReads &R, const Ev &a, const Ev &b) {
    const int64_t sa = R.seq_off[a.read] + a.ridx, sb = R.seq_off[b.read] + b.ridx;
    const int n = min((int) a.klen, (int) b.klen);
    for (int i = 12; i < n; i++) {
        const int ra = nt16_ascii_rank(seq_code_at(R.seq, sa + i)), rb = nt16_ascii_rank(seq_code_at(R.seq, sb + i));
        if (ra != rb) return ra - rb;
    }
    return (int) a.klen - (int) b.klen;
}
__device__ __forceinline__ int allele_cmp(const DevReads &R, const Ev &a, const Ev &b) {
    if (a.type != b.type) return (int) a.type - (int) b.type;
    if (a.key != b.key) return a.key < b.key ? -1 : 1;
    if (a.type == 2 && a.klen > 12 && b.klen > 12) return ins_tail_cmp(R, a, b);
    return (int) a.klen - (int) b.klen;
}

__global__ void k_site_alleles(AlleleArgs A) {
    const int lane = threadIdx.x & 31;
    const int64_t s = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (s >= A.n_sites) return;
    const int64_t g = A.site_g[s];
    const int reg = find_region(A.region_goff, A.n_regions, g);
    const pb_region_t rg = A.regions[reg];
    const int64_t x = g - A.region_goff[reg];
    const uint32_t m = A.meta[g];
    const int64_t e0 = A.site_evoff[s];
    const int n = (int) (A.site_evoff[s + 1] - e0);
    Ev *ev = A.ev + e0;
    const int npseudo = (m & F_SNP) ? 4 : 0;
    const char rch = (x < rg.ref_len) ? A.ref[rg.ref_off + x] : '\0';
    const int rcls = ref_class(rch);
    const int cov = A.cov[g];
    const int depth = min(cov, 125);                                   // region_summary.cpp:682
    const double ddepth = fmax(1.0, (double) depth);
    const VParams &P = A.P;
    if (lane == 0) A.site_region[s] = reg;

    // A. SNP alleles of A/C/G/T read straight from the (unclamped) columns
    if (lane < npseudo) {
        const int code = 1 << lane;                                    // A=1 C=2 G=4 T=8
        Ev v; memset(&v, 0, sizeof(v));
        v.type = 1; v.klen = 1; v.code = (uint8_t) code; v.key = (uint64_t) nt16_ascii_rank(code);
        if (rcls < 4 && nt16_char(code) != rch) {
            const int f = -(int) A.M16[g * 16 + 1 + lane], r = -(int) A.M16[g * 16 + 9 + lane];
            v.total = f + r; v.fwd = f; v.leader = (f + r) > 0;
        }
        ev[lane] = v;
    }
    __syncwarp();
    // B. leaders among the real events
    for (int i = npseudo + lane; i < n; i += 32) {
        const Ev me = ev[i];
        bool lead = true;
        for (int j = npseudo; j < i && lead; j++) if (allele_cmp(A.R, ev[j], me) == 0) lead = false;
        ev[i].leader = lead;
    }
    __syncwarp();
    // C. totals + filters (region_summary.cpp:686-712)
    for (int i = lane; i < n; i += 32) {
        Ev me = ev[i];
        if (!me.leader) { ev[i].pass = 0; continue; }
        if (i >= npseudo) {
            int tot = 0, fwd = 0;
            for (int j = npseudo; j < n; j++) {
                const Ev o = ev[j];
                if (allele_cmp(A.R, o, me) == 0) { tot++; fwd += (o.strand == 0); }
            }
            me.total = tot; me.fwd = fwd;
        }
        const double freq = (double) me.total / ddepth;
        bool pass = true;
        if ((double) me.total < P.support_thr) pass = false;
        if (me.type != 1 && freq < P.indel_cand_thr) pass = false;
        if (me.type == 1 && freq < P.snp_cand_thr) pass = false;
        if (me.type != 1 && P.skip_indels) pass = false;
        if ((me.type == 1 && !(m & F_SNP)) || (me.type == 2 && !(m & F_INS)) || (me.type == 3 && !(m & F_DEL))) pass = false;
        me.pass = pass;
        ev[i] = me;
    }
    __syncwarp();
    // D. order of the passing alleles
    int npass = 0;
    for (int i = lane; i < n; i += 32) {
        const Ev me = ev[i];
        if (!me.pass) continue;
        int ord = 0;
        for (int j = 0; j < n; j++) {
            const Ev o = ev[j];
            if (o.pass && allele_cmp(A.R, o, me) < 0) ord++;
        }
        Cand c; memset(&c, 0, sizeof(c));
        c.read = me.read; c.ridx = me.ridx; c.total = me.total; c.fwd = me.fwd; c.rev = me.total - me.fwd;
        c.klen = me.klen; c.type = me.type; c.code = me.code;
        A.cand_tmp[e0 + ord] = c;
        npass++;
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) npass += __shfl_xor_sync(0xffffffffu, npass, d);
    if (lane == 0) A.site_ncand[s] = npass;
}

// ------------------------------------------------------------------ k_windows
struct WindowArgs {
    DevReads R;
    const pb_region_t *regions;
    const char *ref;
    const int64_t *region_goff;
    const uint32_t *site_g;
    const int64_t *site_evoff;
    const int32_t *site_region;
    const int64_t *site_candoff;     // [n_sites+1]
    const int16_t *M16;
    const int32_t *cov;
    const Cand *cand_tmp;
    int64_t n_sites, capacity;
    int8_t *images; int64_t *positions; uint8_t *depths, *freqs; char *keys; int32_t *region_of;
};

// region_summary.cpp:201-230 for an upper-case class of the reference base
__device__ __forceinline__ int feat_col(int rcls, char base, int rev) {
    if (rcls >= 4) return -1;
    const int start = rev ? 18 : 7;
    switch (to_upper(base)) {
        case 'A': return start + 1; case 'C': return start + 2; case 'G': return start + 3; case 'T': return start + 4;
        case 'I': return start + 5; case 'D': return start + 6; default: return start + 7;
    }
}

// One warp per flagged site.  The 33 x 26 window of the (clamped, int8) base matrix around the site is built ONCE per site in
// shared memory — 33 matrix rows fetched as 16-byte vectors — and every candidate of the site is that window with the few
// candidate cells of row 16 (rows 17.. for a deletion) patched on the way out, stored two bytes per lane.
constexpr int WIN_CELLS = 33 * 26;
// image column j -> column of the 16-wide int16 matrix row (REFF, 7 forward features, REFR, 7 reverse features), -1 = a zero column
__device__ __forceinline__ int win_col(int j) { return j == 4 ? 0 : (j >= 8 && j <= 15) ? j - 7 : j >= 19 ? j - 10 : -1; }

__global__ void __launch_bounds__(128) k_windows(WindowArgs A) {
    __shared__ __align__(16) int16_t s_rows[4][33][16];
    __shared__ __align__(4) int8_t s_base[4][WIN_CELLS + 6];
    __shared__ int8_t s_refc[4][36];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int64_t s = (int64_t) blockIdx.x * (blockDim.x >> 5) + wib;
    if (s >= A.n_sites) return;
    const int64_t o0 = A.site_candoff[s];
    const int nc = (int) (A.site_candoff[s + 1] - o0);
    if (nc == 0) return;
    const int64_t g = A.site_g[s];
    const int reg = A.site_region[s];
    const pb_region_t rg = A.regions[reg];
    const int64_t gbase = A.region_goff[reg];
    const int64_t x = g - gbase;
    const int64_t L1 = rg.ref_end - rg.ref_start + 1;
    const char rch = (x < rg.ref_len) ? A.ref[rg.ref_off + x] : '\0';
    const int rcls = ref_class(rch);
    const int depth = min(A.cov[g], 125);
    // ---- the site's window: rows outside [0, region_size) are zero; row region_size is the spare zero row
    for (int it = lane; it < 66; it += 32) {
        const int i = it >> 1, h = it & 1;
        const int64_t xr = x - 16 + i;
        int4 v = make_int4(0, 0, 0, 0);
        if (xr >= 0 && xr < L1) v = __ldg(reinterpret_cast<const int4 *>(A.M16 + (gbase + xr) * 16 + h * 8));
        *reinterpret_cast<int4 *>(&s_rows[wib][i][h * 8]) = v;
    }
    for (int i = lane; i < 33; i += 32) {                            // column 0: the reference base code of every row
        const int64_t xr = x - 16 + i;
        int v = 0;
        if (xr >= 0 && xr < L1) {
            const char c = (xr < rg.ref_len) ? to_upper(A.ref[rg.ref_off + xr]) : '\0';
            v = c == 'A' ? 1 : c == 'C' ? 2 : c == 'G' ? 3 : c == 'T' ? 4 : 5;
        }
        s_refc[wib][i] = (int8_t) v;
    }
    __syncwarp();
#pragma unroll 9
    for (int e = lane; e < WIN_CELLS; e += 32) {
        const int i = e / 26, j = e - i * 26;
        const int k = win_col(j);
        int v = 0;
        if (j == 0) v = s_refc[wib][i];
        else if (k >= 0) {                                           // rows outside the region were staged as zeros
            v = s_rows[wib][i][k];
            if (j >= 11 && j <= 24) v = v >= 0 ? min(v, 125) : max(v, -125);      // the clamp of :648-653
        }
        s_base[wib][e] = (int8_t) v;                                 // int8 wrap == DataStore.py:68 astype
    }
    __syncwarp();
    const int8_t *base = s_base[wib];
    for (int c = 0; c < nc; c++) {
        const int64_t o = o0 + c;
        if (o >= A.capacity) return;
        const Cand cd = A.cand_tmp[A.site_evoff[s] + c];
        const int klen = cd.klen;
        const int fwd = min(cd.fwd, 125), rev = min(cd.rev, 125);
        char snp_char = 0;
        int ff, fr, sf = -1, sr = -1, end_index = 16;
        if (cd.type == 1) {
            snp_char = nt16_char(cd.code);
            ff = feat_col(rcls, snp_char, 0); fr = feat_col(rcls, snp_char, 1);
        } else if (cd.type == 2) {
            ff = feat_col(rcls, 'I', 0); fr = feat_col(rcls, 'I', 1);
        } else {
            ff = feat_col(rcls, 'D', 0); fr = feat_col(rcls, 'D', 1);
            sf = feat_col(rcls, '*', 0); sr = feat_col(rcls, '*', 1);
            end_index = min(16 + klen - 1, 31);
        }
        const int patch_end = (end_index + 1) * 26;                  // cells [16 * 26, patch_end) may differ from the window
        uint16_t *img = reinterpret_cast<uint16_t *>(A.images + o * WIN_CELLS);        // o * 858 is even
        for (int t = lane; t < WIN_CELLS / 2; t += 32) {
            const int e0 = 2 * t;
            const uint32_t pair = reinterpret_cast<const uint16_t *>(base)[t];
            int v2[2] = {(int) (int8_t) (pair & 0xffu), (int) (int8_t) (pair >> 8)};
            if (e0 + 1 >= 16 * 26 && e0 < patch_end) {
#pragma unroll
                for (int q = 0; q < 2; q++) {
                    const int e = e0 + q;
                    const int i = e / 26, j = e - i * 26;
                    int v = v2[q];
                    if (i == 16) {
                        if (cd.type == 1) {
                            if (j == 1) v = (snp_char == 'A') ? 1 : (snp_char == 'C') ? 2 : (snp_char == 'G') ? 3 : (snp_char == 'T') ? 4 : 5;
                            else if (j == 5) v = fwd; else if (j == 16) v = rev;
                        } else if (cd.type == 2) {
                            if (j == 2) v = min(klen, 125); else if (j == 6) v = fwd; else if (j == 17) v = rev;
                        } else {
                            if (j == 3) v = min(klen, 125); else if (j == 7) v = fwd; else if (j == 18) v = rev;
                        }
                        if (j == ff || j == fr) v = -v;
                    } else if (cd.type == 3 && i > 16 && i <= end_index) {
                        if (j == 3) v = min(klen, 125); else if (j == 7) v = fwd; else if (j == 18) v = rev;
                        if (j == sf || j == sr) v = -v;
                    }
                    v2[q] = v;
                }
            }
            img[t] = (uint16_t) ((uint32_t) (uint8_t) (int8_t) v2[0] | ((uint32_t) (uint8_t) (int8_t) v2[1] << 8));
        }
        // key string, 64 B
        for (int k = lane; k < PB_ALLELE_STRIDE; k += 32) {
            char ch = 0;
            if (k == 0) ch = (char) ('0' + cd.type);
            else if (k <= klen) {
                if (cd.type == 1) ch = snp_char;
                else if (cd.type == 2) ch = nt16_char(seq_code_at(A.R.seq, A.R.seq_off[cd.read] + cd.ridx + (k - 1)));
                else ch = A.ref[rg.ref_off + x + (k - 1)];
            }
            A.keys[o * PB_ALLELE_STRIDE + k] = ch;
        }
        if (lane == 0) {
            A.positions[o] = rg.ref_start + x;
            A.depths[o] = (uint8_t) depth;
            A.freqs[o] = (uint8_t) min(cd.total, 125);
            A.region_of[o] = reg;
        }
    }
}

__global__ void k_region_counts(const int32_t *__restrict__ region_of, int64_t n, int64_t *__restrict__ per_region) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(reinterpret_cast<unsigned long long *>(per_region + region_of[i]), 1ULL);
}

}  // namespace pb

// =====================================================================================================
// host side
// =====================================================================================================
using namespace pb;


extern "C" int pb_variant_encoder_create(pb_variant_encoder_t **out, int device) {
    if (!out) { set_error("null out"); return PB_ERR_ARG; }
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= device) {
        set_error("no CUDA device %d (found %d): libpepper_b200 has no CPU fallback", device, n);
        return PB_ERR_CUDA;
    }
    PB_CUDA(cudaSetDevice(device));
    auto *e = new pb_variant_encoder();
    e->device = device;
    for (auto &ev : e->evt) PB_CUDA(cudaEventCreate(&ev));
    PB_CUDA(cudaFuncSetAttribute(k_tile_count, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int) (NCNT * TILE * sizeof(int32_t) + 2 * TILE)));
    *out = e;
    return PB_OK;
}

extern "C" int pb_variant_encoder_destroy(pb_variant_encoder_t *e) {
    if (!e) return PB_OK;
    DevBuf *bufs[] = {&e->op_ref, &e->op_rd, &e->read_reflen, &e->read_region, &e->tile_region, &e->tile_x0, &e->region_goff,
                      &e->M16, &e->cov, &e->meta, &e->dbg, &e->tile_nsites, &e->tile_nev, &e->tile_site_base,
                      &e->tile_ev_base, &e->site_of, &e->site_g, &e->site_evoff, &e->site_cur, &e->ev, &e->cand_tmp,
                      &e->site_ncand, &e->site_region, &e->site_candoff, &e->rare, &e->scalars,
                      &e->h_pos, &e->h_seq_off, &e->h_cigar_off, &e->h_flags, &e->h_mapq, &e->h_seq, &e->h_qual,
                      &e->h_cigar, &e->h_regions, &e->h_ref, &e->o_images, &e->o_positions, &e->o_depths, &e->o_freqs,
                      &e->o_keys, &e->o_region_of, &e->o_per_region, &e->p_images, &e->p_positions, &e->p_depths, &e->p_freqs,
                      &e->p_keys, &e->p_region_of, &e->p_probs, &e->p_per_region};
    for (auto *b : bufs) b->release();
    for (auto &ev : e->evt) if (ev) cudaEventDestroy(ev);
    for (auto &ev : e->pevt) if (ev) cudaEventDestroy(ev);
    for (int b = 0; b < 2; b++) { for (auto &gb : e->g_buf[b]) gb.release(); if (e->copied[b]) cudaEventDestroy(e->copied[b]); }
    if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
    delete e;
    return PB_OK;
}

extern "C" int pb_variant_encoder_set_debug(pb_variant_encoder_t *e, int on) {
    if (!e) return PB_ERR_ARG;
    e->debug = on != 0;
    return PB_OK;
}

static VParams make_params(const pb_variant_params_t *p) {
    VParams P;
    P.min_snp_baseq = p->min_snp_baseq;
    P.min_indel_baseq = p->min_indel_baseq;
    double c = p->min_snp_baseq;
    long long ci = (long long) c;
    if ((double) ci < c) ci++;                     // ceil
    if (ci < 0) ci = 0;
    if (ci > 256) ci = 256;
    P.minq_snp = (int) ci;
    P.snp_thr = p->snp_freq_threshold; P.ins_thr = p->insert_freq_threshold; P.del_thr = p->delete_freq_threshold;
    P.min_cov = p->min_coverage_threshold; P.snp_cand_thr = p->snp_candidate_freq_threshold;
    P.indel_cand_thr = p->indel_candidate_freq_threshold; P.support_thr = p->candidate_support_threshold;
    P.skip_indels = p->skip_indels;
    return P;
}

extern "C" int pb_variant_encode_device(pb_variant_encoder_t *e, const pb_reads_t *dr, const pb_region_t *d_regions,
                                        int64_t n_regions, const pb_region_t *h_regions, const char *d_ref,
                                        int64_t ref_bytes, const pb_variant_params_t *params, int64_t capacity,
                                        int8_t *d_images, int64_t *d_positions, uint8_t *d_depths, uint8_t *d_freqs,
                                        char *d_keys, int32_t *d_region_of, int64_t *d_n_per_region, int64_t *n_out,
                                        void *stream_) {
    if (!e || !dr || !h_regions || !params || !n_out) { set_error("null argument"); return PB_ERR_ARG; }
    if (reinterpret_cast<uintptr_t>(d_images) & 1) { set_error("d_images must be 2-byte aligned"); return PB_ERR_ARG; }   // k_windows stores pairs
    (void) ref_bytes;
    cudaStream_t st = (cudaStream_t) stream_;
    PB_CUDA(cudaSetDevice(e->device));
    *n_out = 0;
    if (d_n_per_region && n_regions > 0) PB_CUDA(cudaMemsetAsync(d_n_per_region, 0, sizeof(int64_t) * n_regions, st));
    if (n_regions <= 0) return PB_OK;
    const VParams P = make_params(params);
    e->launches = 0;

    // ---- host-side tables: tiles, global position offsets, read -> region
    const int64_t n_reads = dr->n_reads;
    std::vector<int64_t> goff(n_regions + 1, 0);
    std::vector<int32_t> tile_region, tile_x0;
    for (int64_t r = 0; r < n_regions; r++) {
        const int64_t L1 = h_regions[r].ref_end - h_regions[r].ref_start + 1;
        if (L1 <= 0) { set_error("region %lld has ref_end < ref_start", (long long) r); return PB_ERR_ARG; }
        if (h_regions[r].read_begin < 0 || h_regions[r].read_end > n_reads || h_regions[r].read_begin > h_regions[r].read_end) {
            set_error("region %lld read range out of bounds", (long long) r); return PB_ERR_ARG;
        }
        goff[r + 1] = goff[r] + L1;
        for (int64_t x = 0; x < L1; x += TILE) { tile_region.push_back((int32_t) r); tile_x0.push_back((int32_t) x); }
    }
    const int64_t G = goff[n_regions];
    if (G >= (1LL << 32)) { set_error("batch covers %lld positions (limit 2^32): split the call", (long long) G); return PB_ERR_ARG; }
    const int64_t n_tiles = (int64_t) tile_region.size();
    std::vector<int32_t> read_region((size_t) std::max<int64_t>(n_reads, 1), -1);
    for (int64_t r = 0; r < n_regions; r++)
        for (int64_t i = h_regions[r].read_begin; i < h_regions[r].read_end; i++) read_region[i] = (int32_t) r;

    // total ops: last cigar_off (device) -> fetch
    // ops of THIS batch: cigar_off may carry absolute offsets into a larger array (region groups of a streaming session view a
    // resident workload through shifted base pointers), so the per-op prefix arrays are sized by last - first and addressed through
    // a base pointer shifted back by `first` — not by the absolute end, which grew (and re-allocated) with every group
    int64_t op_first = 0, op_last = 0;
    if (n_reads > 0) {
        PB_CUDA(cudaMemcpyAsync(&op_first, dr->cigar_off, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(&op_last, dr->cigar_off + n_reads, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    }
    PB_CUDA(cudaStreamSynchronize(st));
    const int64_t n_ops = op_last - op_first;
    if (n_ops < 0) { set_error("cigar offsets are not ascending"); return PB_ERR_ARG; }

    PB_TRY(e->op_ref.reserve(sizeof(int32_t) * (n_ops + 1)));
    PB_TRY(e->op_rd.reserve(sizeof(int32_t) * (n_ops + 1)));
    int32_t *const op_ref_base = e->op_ref.as<int32_t>() - op_first, *const op_rd_base = e->op_rd.as<int32_t>() - op_first;
    PB_TRY(e->read_reflen.reserve(sizeof(int32_t) * (n_reads + 1)));
    PB_TRY(e->read_region.reserve(sizeof(int32_t) * (n_reads + 1)));
    PB_TRY(e->tile_region.reserve(sizeof(int32_t) * n_tiles));
    PB_TRY(e->tile_x0.reserve(sizeof(int32_t) * n_tiles));
    PB_TRY(e->region_goff.reserve(sizeof(int64_t) * (n_regions + 1)));
    PB_TRY(e->M16.reserve(sizeof(int16_t) * 16 * G));
    PB_TRY(e->cov.reserve(sizeof(int32_t) * G));
    PB_TRY(e->meta.reserve(sizeof(uint32_t) * G));
    PB_TRY(e->site_of.reserve(sizeof(uint32_t) * G));
    if (e->debug) PB_TRY(e->dbg.reserve(sizeof(int32_t) * 3 * G));
    PB_TRY(e->tile_nsites.reserve(sizeof(int32_t) * n_tiles));
    PB_TRY(e->tile_nev.reserve(sizeof(int32_t) * n_tiles));
    PB_TRY(e->tile_site_base.reserve(sizeof(int64_t) * (n_tiles + 1)));
    PB_TRY(e->tile_ev_base.reserve(sizeof(int64_t) * (n_tiles + 1)));
    PB_TRY(e->scalars.reserve(sizeof(int64_t) * 8));
    PB_TRY(e->rare.reserve(sizeof(RareEv) * e->rare_cap));

    PB_CUDA(cudaMemcpyAsync(e->tile_region.p, tile_region.data(), sizeof(int32_t) * n_tiles, cudaMemcpyHostToDevice, st));
    PB_CUDA(cudaMemcpyAsync(e->tile_x0.p, tile_x0.data(), sizeof(int32_t) * n_tiles, cudaMemcpyHostToDevice, st));
    PB_CUDA(cudaMemcpyAsync(e->region_goff.p, goff.data(), sizeof(int64_t) * (n_regions + 1), cudaMemcpyHostToDevice, st));
    if (n_reads > 0)
        PB_CUDA(cudaMemcpyAsync(e->read_region.p, read_region.data(), sizeof(int32_t) * n_reads, cudaMemcpyHostToDevice, st));
    PB_CUDA(cudaMemsetAsync(e->scalars.p, 0, sizeof(int64_t) * 8, st));
    int64_t *sc = e->scalars.as<int64_t>();      // [0] n_sites [1] n_ev [2] rare_n [3] n_cand

    DevReads R{dr->pos, dr->seq_off, dr->cigar_off, dr->flags, dr->mapq, dr->seq, dr->qual, dr->cigar, n_reads};

    PB_CUDA(cudaEventRecord(e->evt[0], st));
    if (n_reads > 0) {
        const int wpb = 8;
        k_cigar_prefix<<<(unsigned) ceil_div(n_reads, wpb), wpb * 32, 0, st>>>(R, op_ref_base, op_rd_base,
                                                                              e->read_reflen.as<int32_t>());
        e->launches++;
    }
    PB_CUDA(cudaEventRecord(e->evt[1], st));

    TileArgs TA;
    TA.R = R; TA.regions = d_regions; TA.ref = d_ref;
    TA.op_ref = op_ref_base; TA.op_rd = op_rd_base; TA.read_reflen = e->read_reflen.as<int32_t>();
    TA.tile_region = e->tile_region.as<int32_t>(); TA.tile_x0 = e->tile_x0.as<int32_t>();
    TA.region_goff = e->region_goff.as<int64_t>();
    TA.M16 = e->M16.as<int16_t>(); TA.cov = e->cov.as<int32_t>(); TA.meta = e->meta.as<uint32_t>();
    TA.dbg_counts = e->debug ? e->dbg.as<int32_t>() : nullptr;
    TA.tile_nsites = e->tile_nsites.as<int32_t>(); TA.tile_nev = e->tile_nev.as<int32_t>();
    TA.rare = e->rare.as<RareEv>(); TA.rare_n = reinterpret_cast<unsigned long long *>(sc + 2); TA.rare_cap = e->rare_cap;
    TA.track = e->track; TA.track_reg = e->track_reg;
    TA.P = P;
    const size_t tc_smem = NCNT * TILE * sizeof(int32_t) + 2 * TILE;
    unsigned long long n_rare = 0;
    for (int attempt = 0; attempt < 2; attempt++) {
        k_tile_count<<<(unsigned) n_tiles, TC_THREADS, tc_smem, st>>>(TA);
        e->launches++;
        PB_CUDA(cudaGetLastError());
        PB_CUDA(cudaMemcpyAsync(&n_rare, sc + 2, sizeof(n_rare), cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        if (n_rare <= e->rare_cap) break;
        // rare-event list overflowed: grow and recount (the counting itself is idempotent)
        e->rare_cap = (size_t) n_rare + (size_t) n_rare / 4 + 1024;
        PB_TRY(e->rare.reserve(sizeof(RareEv) * e->rare_cap));
        TA.rare = e->rare.as<RareEv>(); TA.rare_cap = e->rare_cap;
        PB_CUDA(cudaMemsetAsync(sc + 2, 0, sizeof(int64_t), st));
    }
    PB_CUDA(cudaEventRecord(e->evt[2], st));

    k_scan_excl<<<1, 1024, 0, st>>>(e->tile_nsites.as<int32_t>(), e->tile_site_base.as<int64_t>(), n_tiles, sc + 0);
    k_scan_excl<<<1, 1024, 0, st>>>(e->tile_nev.as<int32_t>(), e->tile_ev_base.as<int64_t>(), n_tiles, sc + 1);
    e->launches += 2;
    int64_t hs[2] = {0, 0};
    PB_CUDA(cudaMemcpyAsync(hs, sc, sizeof(int64_t) * 2, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    const int64_t n_sites = hs[0], n_ev = hs[1];

    e->last_goff = goff;
    e->last_regions.assign(h_regions, h_regions + n_regions);
    e->last_d_ref = d_ref;

    int64_t n_cand = 0;
    if (n_sites > 0) {
        PB_TRY(e->site_g.reserve(sizeof(uint32_t) * n_sites));
        PB_TRY(e->site_evoff.reserve(sizeof(int64_t) * (n_sites + 1)));
        PB_TRY(e->site_cur.reserve(sizeof(uint32_t) * n_sites));
        PB_TRY(e->site_ncand.reserve(sizeof(int32_t) * n_sites));
        PB_TRY(e->site_region.reserve(sizeof(int32_t) * n_sites));
        PB_TRY(e->site_candoff.reserve(sizeof(int64_t) * (n_sites + 1)));
        PB_TRY(e->ev.reserve(sizeof(Ev) * (n_ev + 1)));
        PB_TRY(e->cand_tmp.reserve(sizeof(Cand) * (n_ev + 1)));
        PB_CUDA(cudaMemsetAsync(e->site_cur.p, 0, sizeof(uint32_t) * n_sites, st));

        SiteArgs SA;
        SA.regions = d_regions; SA.tile_region = TA.tile_region; SA.tile_x0 = TA.tile_x0; SA.region_goff = TA.region_goff;
        SA.meta = TA.meta; SA.tile_site_base = e->tile_site_base.as<int64_t>(); SA.tile_ev_base = e->tile_ev_base.as<int64_t>();
        SA.site_of = e->site_of.as<uint32_t>(); SA.site_g = e->site_g.as<uint32_t>(); SA.site_evoff = e->site_evoff.as<int64_t>();
        SA.n_sites_total = n_sites; SA.n_ev_total = n_ev;
        k_site_index<<<(unsigned) n_tiles, TILE, 0, st>>>(SA);
        e->launches++;
        PB_CUDA(cudaEventRecord(e->evt[3], st));

        CollectArgs CA;
        CA.R = R; CA.regions = d_regions; CA.read_region = e->read_region.as<int32_t>(); CA.region_goff = TA.region_goff;
        CA.op_ref = TA.op_ref; CA.op_rd = TA.op_rd; CA.meta = TA.meta; CA.site_of = SA.site_of; CA.site_evoff = SA.site_evoff;
        CA.site_cur = e->site_cur.as<uint32_t>(); CA.ev = e->ev.as<Ev>(); CA.rare = e->rare.as<RareEv>(); CA.n_rare = n_rare;
        CA.P = P; CA.op_first = op_first; CA.op_last = op_last;
        if (n_ops > 0) { k_collect_ops<<<(unsigned) ceil_div(n_ops, (int64_t) 8 * COLLECT_CHUNK), 256, 0, st>>>(CA); e->launches++; }
        if (n_rare > 0) { k_collect_rare<<<(unsigned) ceil_div((int64_t) n_rare, 256), 256, 0, st>>>(CA); e->launches++; }

        AlleleArgs AA;
        AA.R = R; AA.regions = d_regions; AA.ref = d_ref; AA.region_goff = TA.region_goff; AA.n_regions = n_regions;
        AA.site_g = SA.site_g; AA.site_evoff = SA.site_evoff; AA.M16 = TA.M16; AA.cov = TA.cov; AA.meta = TA.meta;
        AA.ev = CA.ev; AA.cand_tmp = e->cand_tmp.as<Cand>(); AA.site_ncand = e->site_ncand.as<int32_t>();
        AA.site_region = e->site_region.as<int32_t>(); AA.n_sites = n_sites; AA.P = P;
        k_site_alleles<<<(unsigned) ceil_div(n_sites, 4), 128, 0, st>>>(AA);
        k_scan_excl<<<1, 1024, 0, st>>>(AA.site_ncand, e->site_candoff.as<int64_t>(), n_sites, sc + 3);
        e->launches += 2;
        PB_CUDA(cudaMemcpyAsync(&n_cand, sc + 3, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        PB_CUDA(cudaEventRecord(e->evt[4], st));

        *n_out = n_cand;
        if (n_cand > capacity) {
            PB_CUDA(cudaEventRecord(e->evt[5], st));
            set_error("candidate capacity %lld < %lld needed", (long long) capacity, (long long) n_cand);
            return PB_ERR_CAPACITY;
        }
        if (n_cand > 0) {
            WindowArgs WA;
            WA.R = R; WA.regions = d_regions; WA.ref = d_ref; WA.region_goff = TA.region_goff; WA.site_g = SA.site_g;
            WA.site_evoff = SA.site_evoff; WA.site_region = AA.site_region; WA.site_candoff = e->site_candoff.as<int64_t>();
            WA.M16 = TA.M16; WA.cov = TA.cov; WA.cand_tmp = AA.cand_tmp; WA.n_sites = n_sites; WA.capacity = capacity;
            WA.images = d_images; WA.positions = d_positions; WA.depths = d_depths; WA.freqs = d_freqs; WA.keys = d_keys;
            WA.region_of = d_region_of;
            k_windows<<<(unsigned) ceil_div(n_sites, 4), 128, 0, st>>>(WA);
            e->launches++;
            if (d_n_per_region)
            { k_region_counts<<<(unsigned) ceil_div(n_cand, 256), 256, 0, st>>>(d_region_of, n_cand, d_n_per_region); e->launches++; }
        }
        PB_CUDA(cudaEventRecord(e->evt[5], st));
    } else {
        PB_CUDA(cudaEventRecord(e->evt[3], st));
        PB_CUDA(cudaEventRecord(e->evt[4], st));
        PB_CUDA(cudaEventRecord(e->evt[5], st));
    }
    PB_CUDA(cudaGetLastError());
    PB_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < 5; i++) cudaEventElapsedTime(&e->ms[i], e->evt[i], e->evt[i + 1]);
    return PB_OK;
}

extern "C" int pb_variant_encoder_launches(pb_variant_encoder_t *e, int64_t *n) {
    if (!e || !n) return PB_ERR_ARG;
    *n = e->launches;
    return PB_OK;
}

extern "C" int pb_variant_encoder_timings(pb_variant_encoder_t *e, float *ms5) {
    if (!e || !ms5) return PB_ERR_ARG;
    for (int i = 0; i < 5; i++) ms5[i] = e->ms[i];
    return PB_OK;
}

namespace pb {
int upload(DevBuf &b, const void *h, size_t bytes, cudaStream_t st) {
    PB_TRY(b.reserve(bytes + 16));
    if (bytes) PB_CUDA(cudaMemcpyAsync(b.p, h, bytes, cudaMemcpyHostToDevice, st));
    return PB_OK;
}
}  // namespace pb

// shared with the polish encoder: copy a host read batch to device staging buffers
namespace pb {
int upload_reads(const pb_reads_t *h, DevBuf *const bufs[8], pb_reads_t *d, cudaStream_t st) {
    const int64_t n = h->n_reads;
    const int64_t nb = n ? h->seq_off[n] : 0, nc = n ? h->cigar_off[n] : 0;
    PB_TRY(upload(*bufs[0], h->pos, sizeof(int64_t) * n, st));
    PB_TRY(upload(*bufs[1], h->seq_off, sizeof(int64_t) * (n + 1), st));
    PB_TRY(upload(*bufs[2], h->cigar_off, sizeof(int64_t) * (n + 1), st));
    PB_TRY(upload(*bufs[3], h->flags, n, st));
    PB_TRY(upload(*bufs[4], h->mapq, n, st));
    PB_TRY(upload(*bufs[5], h->seq, (size_t) ((nb + 1) / 2), st));
    PB_TRY(upload(*bufs[6], h->qual, (size_t) nb, st));
    PB_TRY(upload(*bufs[7], h->cigar, sizeof(uint32_t) * nc, st));
    d->n_reads = n;
    d->pos = bufs[0]->as<int64_t>(); d->seq_off = bufs[1]->as<int64_t>(); d->cigar_off = bufs[2]->as<int64_t>();
    d->flags = bufs[3]->as<uint8_t>(); d->mapq = bufs[4]->as<uint8_t>(); d->seq = bufs[5]->as<uint8_t>();
    d->qual = bufs[6]->as<uint8_t>(); d->cigar = bufs[7]->as<uint32_t>();
    return PB_OK;
}
}  // namespace pb

extern "C" int pb_variant_encode_host(pb_variant_encoder_t *e, const pb_reads_t *h_reads, const pb_region_t *h_regions,
                                      int64_t n_regions, const char *h_ref, int64_t ref_bytes,
                                      const pb_variant_params_t *params, int64_t capacity, int8_t *h_images,
                                      int64_t *h_positions, uint8_t *h_depths, uint8_t *h_freqs, char *h_keys,
                                      int32_t *h_region_of, int64_t *h_n_per_region, int64_t *n_out, void *stream_) {
    if (!e || !h_reads || !h_regions || !params || !n_out) { set_error("null argument"); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    PB_CUDA(cudaSetDevice(e->device));
    DevBuf *rb[8] = {&e->h_pos, &e->h_seq_off, &e->h_cigar_off, &e->h_flags, &e->h_mapq, &e->h_seq, &e->h_qual, &e->h_cigar};
    pb_reads_t d;
    int rc = upload_reads(h_reads, rb, &d, st);
    if (rc != PB_OK) return rc;
    PB_TRY(upload(e->h_regions, h_regions, sizeof(pb_region_t) * n_regions, st));
    PB_TRY(upload(e->h_ref, h_ref, (size_t) ref_bytes, st));
    const int64_t cap = std::max<int64_t>(capacity, 1);
    PB_TRY(e->o_images.reserve((size_t) cap * 33 * 26));
    PB_TRY(e->o_positions.reserve(sizeof(int64_t) * cap));
    PB_TRY(e->o_depths.reserve(cap));
    PB_TRY(e->o_freqs.reserve(cap));
    PB_TRY(e->o_keys.reserve((size_t) cap * PB_ALLELE_STRIDE));
    PB_TRY(e->o_region_of.reserve(sizeof(int32_t) * cap));
    PB_TRY(e->o_per_region.reserve(sizeof(int64_t) * std::max<int64_t>(n_regions, 1)));
    rc = pb_variant_encode_device(e, &d, e->h_regions.as<pb_region_t>(), n_regions, h_regions, e->h_ref.as<char>(), ref_bytes,
                                  params, capacity, e->o_images.as<int8_t>(), e->o_positions.as<int64_t>(),
                                  e->o_depths.as<uint8_t>(), e->o_freqs.as<uint8_t>(), e->o_keys.as<char>(),
                                  e->o_region_of.as<int32_t>(), e->o_per_region.as<int64_t>(), n_out, stream_);
    if (rc != PB_OK) return rc;
    const int64_t n = *n_out;
    if (n > 0) {
        PB_CUDA(cudaMemcpyAsync(h_images, e->o_images.p, (size_t) n * 33 * 26, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_positions, e->o_positions.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_depths, e->o_depths.p, n, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_freqs, e->o_freqs.p, n, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_keys, e->o_keys.p, (size_t) n * PB_ALLELE_STRIDE, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_region_of, e->o_region_of.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    }
    if (h_n_per_region && n_regions > 0)
        PB_CUDA(cudaMemcpyAsync(h_n_per_region, e->o_per_region.p, sizeof(int64_t) * n_regions, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    return PB_OK;
}

extern "C" int pb_variant_encoder_debug_region(pb_variant_encoder_t *e, int64_t region, int32_t *h_matrix, int32_t *h_coverage,
                                               int32_t *h_snp, int32_t *h_ins, int32_t *h_del) {
    if (!e || region < 0 || region >= (int64_t) e->last_regions.size()) { set_error("bad region"); return PB_ERR_ARG; }
    const pb_region_t &rg = e->last_regions[region];
    const int64_t L1 = rg.ref_end - rg.ref_start + 1, g0 = e->last_goff[region];
    std::vector<int16_t> m16((size_t) L1 * 16);
    std::vector<char> ref((size_t) std::max<int64_t>(rg.ref_len, 1));
    PB_CUDA(cudaMemcpy(m16.data(), e->M16.as<int16_t>() + g0 * 16, sizeof(int16_t) * 16 * L1, cudaMemcpyDeviceToHost));
    if (rg.ref_len > 0) PB_CUDA(cudaMemcpy(ref.data(), e->last_d_ref + rg.ref_off, (size_t) rg.ref_len, cudaMemcpyDeviceToHost));
    if (h_matrix) {
        for (int64_t x = 0; x < L1; x++) {
            int32_t *row = h_matrix + x * 26;
            for (int j = 0; j < 26; j++) row[j] = 0;
            char c = x < rg.ref_len ? ref[x] : '\0';
            if (c >= 'a' && c <= 'z') c = (char) (c - 32);
            row[0] = c == 'A' ? 1 : c == 'C' ? 2 : c == 'G' ? 3 : c == 'T' ? 4 : 5;
            const int16_t *s = &m16[(size_t) x * 16];
            row[4] = s[0]; row[15] = s[8];
            for (int k = 0; k < 7; k++) { row[8 + k] = s[1 + k]; row[19 + k] = s[9 + k]; }
            for (int j = 11; j < 25; j++) row[j] = row[j] >= 0 ? std::min(row[j], 125) : std::max(row[j], -125);
        }
    }
    if (h_coverage) PB_CUDA(cudaMemcpy(h_coverage, e->cov.as<int32_t>() + g0, sizeof(int32_t) * L1, cudaMemcpyDeviceToHost));
    if (h_snp || h_ins || h_del) {
        if (!e->debug) { set_error("call pb_variant_encoder_set_debug(enc,1) before encoding to keep the count vectors"); return PB_ERR_STATE; }
        std::vector<int32_t> d((size_t) L1 * 3);
        PB_CUDA(cudaMemcpy(d.data(), e->dbg.as<int32_t>() + g0 * 3, sizeof(int32_t) * 3 * L1, cudaMemcpyDeviceToHost));
        for (int64_t x = 0; x < L1; x++) {
            if (h_snp) h_snp[x] = d[x * 3];
            if (h_ins) h_ins[x] = d[x * 3 + 1];
            if (h_del) h_del[x] = d[x * 3 + 2];
        }
    }
    return PB_OK;
}
