// VCF text on the GPU: the site assembly of VCFWriter.candidate_list_to_variant / write_vcf_records
// (pepper_variant/modules/python/VcfWriter.py:48-218, restated on the host by pepper_b200/vcf.py assemble_sites) and the
// data lines pysam writes for those records (vcf.format_vcf_line), one thread per (contig, position) site.
//
//   selection (k_find_candidates) -> stable radix sort by (contig, position) -> site starts -> pass 1: exact line lengths
//   -> exclusive scan -> pass 2: the text, straight into the caller's buffer.
// Both passes run the same device function, so the size pass and the write pass cannot disagree.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace pb {

constexpr int VCF_MAX_ALLELES = 16;            // allowed_multiallelics upper bound (the reference's default is 4)
constexpr int VAF_STRIDE = 8;                  // one NUL-padded "%g" text per (AD, DP) in the VAF table
constexpr uint8_t F_DV = 2, F_REPEAT = 4, F_SWAP = 8;

// ------------------------------------------------------------------ "%.6g" of a float32, exact
// Python's "%.6g" % float(np.float32(x)): six significant digits of the EXACT binary value, round-half-even, then %g's choice
// of fixed or exponent form.  A float32 is m * 2^e (m < 2^24, -149 <= e <= 104); m * 10^k * 2^e for k <= 50 stays below
// 2^192, so six 32-bit limbs hold every intermediate and no floating-point rounding enters the digits.
struct U192 {
    uint32_t w[6];
    __host__ __device__ void set(uint64_t v) { for (int i = 0; i < 6; i++) w[i] = 0; w[0] = (uint32_t) v; w[1] = (uint32_t) (v >> 32); }
    __host__ __device__ void mul10() {
        uint64_t c = 0;
        for (int i = 0; i < 6; i++) { const uint64_t t = (uint64_t) w[i] * 10u + c; w[i] = (uint32_t) t; c = t >> 32; }
    }
    __host__ __device__ uint32_t div10() {                     // returns the remainder
        uint64_t r = 0;
        for (int i = 5; i >= 0; i--) { const uint64_t t = (r << 32) | w[i]; w[i] = (uint32_t) (t / 10u); r = t % 10u; }
        return (uint32_t) r;
    }
    __host__ __device__ bool bit(int b) const { return b >= 0 && b < 192 && ((w[b >> 5] >> (b & 31)) & 1u); }
    __host__ __device__ bool any_below(int b) const {          // any of bits [0, b)
        for (int i = 0; i < 6 && 32 * i < b; i++) {
            const int n = b - 32 * i;
            const uint32_t m = n >= 32 ? 0xffffffffu : ((1u << n) - 1u);
            if (w[i] & m) return true;
        }
        return false;
    }
    __host__ __device__ void shl(int s) { for (int k = 0; k < s; k++) { for (int i = 5; i > 0; i--) w[i] = (w[i] << 1) | (w[i - 1] >> 31); w[0] <<= 1; } }
    __host__ __device__ void shr(int s) {
        const int q = s >> 5, r = s & 31;
        for (int i = 0; i < 6; i++) {
            const uint32_t lo = (i + q < 6) ? w[i + q] : 0u, hi = (i + q + 1 < 6) ? w[i + q + 1] : 0u;
            w[i] = r ? ((lo >> r) | (hi << (32 - r))) : lo;
        }
    }
    __host__ __device__ bool fits64() const { return !(w[2] | w[3] | w[4] | w[5]); }
    __host__ __device__ uint64_t lo64() const { return (uint64_t) w[0] | ((uint64_t) w[1] << 32); }
};

// floor(m * 2^e * 10^k) and where the dropped part lies against one half: 0 below, 1 exactly half, 2 above
__host__ __device__ static uint64_t scaled_floor(uint32_t m, int e, int k, int *half) {
    U192 p; p.set(m);
    if (e > 0) p.shl(e);
    for (int i = 0; i < k; i++) p.mul10();
    bool top = false, sticky = false;                          // most significant dropped digit / bit, and anything below it
    if (e < 0) { top = p.bit(-e - 1); sticky = p.any_below(-e - 1); p.shr(-e); }
    if (k < 0) {
        uint32_t d = 0;
        sticky = sticky || top;
        for (int i = 0; i < -k; i++) { sticky = sticky || d != 0; d = p.div10(); }
        *half = d > 5 || (d == 5 && sticky) ? 2 : d == 5 ? 1 : 0;
    } else {
        *half = top ? (sticky ? 2 : 1) : 0;
    }
    return p.fits64() ? p.lo64() : ~0ull;
}

// writes the text (no NUL) to out when out != nullptr; returns its length (at most 13)
__host__ __device__ int format_g6(float xf, char *out) {
    uint32_t bits;
    memcpy(&bits, &xf, 4);
    char buf[16];
    int n = 0;
    if (bits >> 31) buf[n++] = '-';
    const int be = (int) ((bits >> 23) & 255u);
    const uint32_t man = bits & 0x7fffffu;
    if (be == 255) {
        const char *t = man ? "nan" : "inf";
        if (man) n = 0;
        for (int i = 0; i < 3; i++) buf[n++] = t[i];
    } else if (be == 0 && man == 0) {
        buf[n++] = '0';
    } else {
        const uint32_t m = be ? (man | 0x800000u) : man;
        const int e = be ? be - 150 : -149;
        int X = (int) floor(log10((double) m) + e * 0.30102999566398120);      // decimal exponent; corrected exactly below
        uint64_t q = 0;
        int half = 0;
        for (;;) {
            q = scaled_floor(m, e, 5 - X, &half);
            if (q >= 1000000ull) X++;
            else if (q < 100000ull) X--;
            else break;
        }
        if (half == 2 || (half == 1 && (q & 1))) q++;
        if (q == 1000000ull) { q = 100000ull; X++; }
        char d[6];
        for (int i = 5; i >= 0; i--) { d[i] = (char) ('0' + q % 10); q /= 10; }
        int last = 5;                                          // last significant digit kept after stripping zeros
        while (last > 0 && d[last] == '0') last--;
        if (X < -4 || X >= 6) {
            buf[n++] = d[0];
            if (last > 0) { buf[n++] = '.'; for (int i = 1; i <= last; i++) buf[n++] = d[i]; }
            buf[n++] = 'e';
            buf[n++] = X < 0 ? '-' : '+';
            const int ax = X < 0 ? -X : X;
            if (ax >= 100) buf[n++] = (char) ('0' + ax / 100);
            buf[n++] = (char) ('0' + (ax / 10) % 10);
            buf[n++] = (char) ('0' + ax % 10);
        } else if (X >= 0) {
            for (int i = 0; i <= X; i++) buf[n++] = d[i];
            if (last > X) { buf[n++] = '.'; for (int i = X + 1; i <= last; i++) buf[n++] = d[i]; }
        } else {
            buf[n++] = '0'; buf[n++] = '.';
            for (int i = 0; i < -X - 1; i++) buf[n++] = '0';
            for (int i = 0; i <= last; i++) buf[n++] = d[i];
        }
    }
    if (out) for (int i = 0; i < n; i++) out[i] = buf[i];
    return n;
}

// QUAL = max(1, int(-10 log10(max(1e-9, 1 - p)))) (VcfWriter.py:156); the clamp is the constant 90, exactly as Python prints it
__device__ int vcf_qual(float p) {
    const double x = 1.0 - (double) p;
    return x > 1e-9 ? max(1, (int) (-10.0 * log10(x))) : 90;
}

// ------------------------------------------------------------------ site assembly + text
struct VcfArgs {
    const int64_t *pos; const int32_t *rof; const uint8_t *dep, *frq; const char *keys; const float *probs;
    const uint8_t *flags, *geno;
    const pb_region_t *regions; const char *ref;
    const int32_t *contig_of_region; const char *names; const int64_t *name_off;
    const char *vaf_table;                                     // [256][256][VAF_STRIDE]: "%g" of round(ad / max(1, dp), 3)
    const int64_t *order;                                      // record indices sorted (stably) by (contig, position)
    const int64_t *site_start;                                 // [n_sites + 1] into order
    int64_t n_sites;
    pb_vcf_options_t O;
};

struct Cursor {                                                // counts always, writes when p != nullptr
    char *p; int64_t n;
    __device__ void put(char c) { if (p) p[n] = c; n++; }
    __device__ void put(const char *s, int len) { if (p) for (int i = 0; i < len; i++) p[n + i] = s[i]; n += len; }
    __device__ void cstr(const char *s) { while (*s) put(*s++); }
    __device__ void u64(uint64_t v) {
        char t[20]; int k = 0;
        do { t[k++] = (char) ('0' + v % 10); v /= 10; } while (v);
        while (k) put(t[--k]);
    }
    __device__ void g6(float x) { n += format_g6(x, p ? p + n : nullptr); }
};

__device__ __forceinline__ int key_len(const char *key) {     // length of the allele key[1:]
    int k = 1;
    while (k < PB_ALLELE_STRIDE && key[k]) k++;
    return k - 1;
}

// ranking of VcfWriter.py:49: (genotype, genotype probability) descending, ties in arrival order (the sort is stable)
__device__ __forceinline__ bool ranks_before(int g1, float p1, int64_t j1, int g2, float p2, int64_t j2) {
    return g1 != g2 ? g1 > g2 : p1 != p2 ? p1 > p2 : j1 < j2;
}

// One site: the line's length (0 = no line); with `out`, the text and the line table entry.
__device__ int64_t site_line(const VcfArgs &A, int64_t s, char *out, pb_vcf_line_t *line) {
    const int64_t a = A.site_start[s], b = A.site_start[s + 1];
    const int64_t i0 = A.order[a];
    if (!(A.flags[i0] & F_DV)) return 0;                      // non-selected records sort last, as one key
    const pb_region_t rg0 = A.regions[A.rof[i0]];
    const int64_t p = A.pos[i0];
    const char rb = to_upper(A.ref[rg0.ref_off + p - rg0.ref_start]);
    // (ref, alt) of the record at sorted index j: the 1-base allele is the reference base
    auto allele = [&](int64_t j, bool want_ref, const char **ptr) -> int {
        const int64_t i = A.order[j];
        const bool swap = (A.flags[i] & F_SWAP) != 0;
        if (want_ref != swap) { *ptr = &rb; return 1; }
        *ptr = A.keys + i * PB_ALLELE_STRIDE + 1;
        return key_len(A.keys + i * PB_ALLELE_STRIDE);
    };
    auto same = [&](int64_t j1, int64_t j2) -> bool {
        for (int w = 0; w < 2; w++) {
            const char *x, *y;
            const int nx = allele(j1, w == 0, &x), ny = allele(j2, w == 0, &y);
            if (nx != ny) return false;
            for (int k = 0; k < nx; k++) if (x[k] != y[k]) return false;
        }
        return true;
    };
    // kept = selected and the first record of its (ref, alt) at this site (CandidateFinder.py:547-574)
    auto kept = [&](int64_t j) -> bool {
        if (!(A.flags[A.order[j]] & F_DV)) return false;
        for (int64_t t = a; t < j; t++) if ((A.flags[A.order[t]] & F_DV) && same(t, j)) return false;
        return true;
    };
    auto pv = [&](int64_t j) -> float { const int64_t i = A.order[j]; return A.probs[i * 3 + A.geno[i]]; };
    // the best allowed_multiallelics records in rank order: each pick is the best one ranked after the previous pick
    int64_t sel[VCF_MAX_ALLELES];
    int m = 0;
    for (; m < A.O.allowed_multiallelics; m++) {
        int64_t best = -1;
        for (int64_t j = a; j < b; j++) {
            if (!kept(j)) continue;
            const int g = A.geno[A.order[j]];
            if (m > 0 && !ranks_before(A.geno[A.order[sel[m - 1]]], pv(sel[m - 1]), sel[m - 1], g, pv(j), j)) continue;
            if (best < 0 || ranks_before(g, pv(j), j, A.geno[A.order[best]], pv(best), best)) best = j;
        }
        if (best < 0) break;
        sel[m] = best;
    }
    if (m == 0) return 0;
    // site values (VcfWriter.py:53-135)
    int longest = 0, max_rlen = 0, n_het = 0, n_hom = 0, depth = 0;
    bool rep = false;
    float gt_qual = -1.f;
    for (int t = 0; t < m; t++) {
        const int64_t i = A.order[sel[t]];
        const char *r;
        const int rl = allele(sel[t], true, &r);
        if (rl > max_rlen) { max_rlen = rl; longest = t; }
        const int g = A.geno[i];
        n_het += g == 1; n_hom += g == 2;
        depth = t ? min(depth, (int) A.dep[i]) : (int) A.dep[i];
        rep = rep || (A.flags[i] & F_REPEAT);
        if (g != 0) gt_qual = gt_qual < 0.f ? pv(sel[t]) : fminf(gt_qual, pv(sel[t]));
        else if (gt_qual < 0.f) gt_qual = fmaxf(A.probs[i * 3 + 1], A.probs[i * 3 + 2]);
    }
    const char *lref;
    allele(sel[longest], true, &lref);
    int gt0 = 0, gt1 = 0;                                      // 0 < hp1 + hp2 <= 2 (VcfWriter.py:130-135); hom-alt ranks first
    if (n_hom == 1 && n_het == 0) { gt0 = 1; gt1 = 1; }
    else if (n_hom == 0 && n_het == 1) { gt1 = 1; }
    else if (n_hom == 0 && n_het == 2) { gt0 = 1; gt1 = 2; }
    const int qual = vcf_qual(gt_qual);
    bool snp = max_rlen == 1;
    for (int t = 0; t < m && snp; t++) {
        const char *al, *rl_;
        snp = allele(sel[t], false, &al) + max_rlen - allele(sel[t], true, &rl_) == 1;
    }
    const double cut = snp ? (rep ? A.O.snp_q_cutoff_in_lc : A.O.snp_q_cutoff) : (rep ? A.O.indel_q_cutoff_in_lc : A.O.indel_q_cutoff);
    const bool refcall = gt0 == 0 && gt1 == 0;
    const bool regenotype = refcall || qual <= cut;

    // CHROM POS ID REF ALT QUAL FILTER INFO FORMAT SAMPLE  (GT:AP:GQ:DP:AD:VAF:REP)
    const int32_t contig = A.contig_of_region[A.rof[i0]];
    Cursor c{out, 0};
    c.put(A.names + A.name_off[contig], (int) (A.name_off[contig + 1] - A.name_off[contig]));
    c.put('\t'); c.u64((uint64_t) p + 1); c.cstr("\t.\t");
    {
        const char *r0;
        const int n0 = allele(sel[0], true, &r0);
        c.put(r0, n0); c.put(lref + n0, max_rlen - n0);
    }
    c.put('\t');
    for (int t = 0; t < m; t++) {
        const char *al, *r;
        const int na = allele(sel[t], false, &al), nr = allele(sel[t], true, &r);
        if (t) c.put(',');
        c.put(al, na); c.put(lref + nr, max_rlen - nr);
    }
    c.put('\t'); c.u64((uint64_t) qual);
    c.cstr(refcall ? "\trefCall\t.\tGT:AP:GQ:DP:AD:VAF:REP\t" : "\tPASS\t.\tGT:AP:GQ:DP:AD:VAF:REP\t");
    c.put((char) ('0' + gt0)); c.put('/'); c.put((char) ('0' + gt1)); c.put(':');
    for (int t = 0; t < m; t++) {
        const int64_t i = A.order[sel[t]];
        if (t) c.put(',');
        c.g6(fmaxf(A.probs[i * 3 + 1], A.probs[i * 3 + 2]));
    }
    c.put(':'); c.u64((uint64_t) qual); c.put(':'); c.u64((uint64_t) depth); c.put(':');
    for (int t = 0; t < m; t++) { if (t) c.put(','); c.u64(A.frq[A.order[sel[t]]]); }
    c.put(':');
    for (int t = 0; t < m; t++) {
        if (t) c.put(',');
        const char *v = A.vaf_table + ((size_t) A.frq[A.order[sel[t]]] * 256 + depth) * VAF_STRIDE;
        int k = 0;
        while (k < VAF_STRIDE && v[k]) k++;
        c.put(v, k);
    }
    c.put(':'); c.put(rep ? '1' : '0'); c.put('\n');
    if (line) {
        line->pos = p; line->contig = contig; line->ref_len = max_rlen;
        line->cls = regenotype ? (snp ? PB_VCF_CLASS_VC_SNP : PB_VCF_CLASS_VC_INDEL) : PB_VCF_CLASS_PEPPER;
        line->text_len = (int32_t) c.n;
    }
    return c.n;
}

__global__ void k_site_keys(const int64_t *__restrict__ pos, const int32_t *__restrict__ rof, const int32_t *__restrict__ contig_of_region,
                            const int64_t *__restrict__ window, uint8_t *__restrict__ flags, int64_t n, int64_t *__restrict__ key,
                            int64_t *__restrict__ iota) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    // a record outside its region's window counts as not selected, so the INT64_MAX site it joins still writes no line
    if (window && (pos[i] < window[2 * rof[i]] || pos[i] > window[2 * rof[i] + 1])) flags[i] &= (uint8_t) ~F_DV;
    key[i] = (flags[i] & F_DV) ? (((int64_t) contig_of_region[rof[i]] << 40) | pos[i]) : INT64_MAX;
    iota[i] = i;
}

__global__ void k_gather_lines(const char *__restrict__ text, const pb_vcf_line_t *__restrict__ lines, const int64_t *__restrict__ sel,
                               const int64_t *__restrict__ dst, int64_t n, uint8_t *__restrict__ out) {
    const int64_t w = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;     // one warp per line
    const int lane = threadIdx.x & 31;
    if (w >= n) return;
    const pb_vcf_line_t ln = lines[sel[w]];
    const char *s = text + ln.text_off;
    uint8_t *d = out + dst[w];
    for (int k = lane; k < ln.text_len; k += 32) d[k] = (uint8_t) s[k];
}

__global__ void k_site_heads(const int64_t *__restrict__ key, int64_t n, int32_t *__restrict__ head) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) head[i] = (i == 0 || key[i] != key[i - 1]) ? 1 : 0;
}

__global__ void k_site_starts(const int32_t *__restrict__ head, const int64_t *__restrict__ rank, int64_t n, int64_t *__restrict__ start) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && head[i]) start[rank[i]] = i;
    if (i == 0) start[rank[n]] = n;
}

__global__ void k_site_sizes(VcfArgs A, int32_t *__restrict__ len, int32_t *__restrict__ has) {
    const int64_t s = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= A.n_sites) return;
    const int64_t l = site_line(A, s, nullptr, nullptr);
    len[s] = (int32_t) l;
    has[s] = l > 0;
}

__global__ void k_site_write(VcfArgs A, const int64_t *__restrict__ off, const int64_t *__restrict__ line_of, char *__restrict__ text,
                             pb_vcf_line_t *__restrict__ lines) {
    const int64_t s = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= A.n_sites || line_of[s + 1] == line_of[s]) return;
    pb_vcf_line_t *ln = lines + line_of[s];
    site_line(A, s, text + off[s], ln);
    ln->text_off = off[s];
}

__global__ void k_vcf_qual(const float *__restrict__ p, int64_t n, int32_t *__restrict__ q) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) q[i] = vcf_qual(p[i]);
}

__global__ void k_format_g(const float *__restrict__ x, int64_t n, char *__restrict__ out) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    char *o = out + i * 16;
    const int k = format_g6(x[i], o);
    for (int j = k; j < 16; j++) o[j] = 0;
}

}  // namespace pb

using namespace pb;

extern "C" int pb_variant_vcf_device(const pb_candidate_columns_t *cols, const float *d_probs, int64_t n, const pb_region_t *d_regions,
                                     const char *d_ref, const pb_vcf_job_t *job, const pb_candidate_options_t *sel_opt,
                                     const pb_vcf_options_t *vcf_opt, char *d_text, int64_t text_cap, pb_vcf_line_t *d_lines,
                                     int64_t lines_cap, int64_t *n_text, int64_t *n_lines, void *stream_) {
    if (!cols || !job || !sel_opt || !vcf_opt || !n_text || !n_lines) { set_error("null argument"); return PB_ERR_ARG; }
    if (vcf_opt->allowed_multiallelics < 1 || vcf_opt->allowed_multiallelics > VCF_MAX_ALLELES) {
        set_error("allowed_multiallelics must be in [1, %d]", VCF_MAX_ALLELES); return PB_ERR_ARG;
    }
    *n_text = 0; *n_lines = 0;
    if (n <= 0) return PB_OK;
    cudaStream_t st = (cudaStream_t) stream_;
    DevBuf flags, geno, key, key2, idx, order, head, rank, start, len, has, off, line_of, tmp;
    int rc = PB_OK;
    auto run = [&]() -> int {
        PB_TRY(flags.reserve(n)); PB_TRY(geno.reserve(n));
        PB_TRY(pb_variant_find_candidates_device(cols->positions, cols->region_of, cols->depths, cols->freqs, cols->keys, d_probs, n,
                                                 d_regions, d_ref, sel_opt, flags.as<uint8_t>(), geno.as<uint8_t>(), stream_));
        PB_TRY(key.reserve(8 * n)); PB_TRY(key2.reserve(8 * n)); PB_TRY(idx.reserve(8 * n)); PB_TRY(order.reserve(8 * n));
        const unsigned gb = (unsigned) ceil_div(n, 256);
        k_site_keys<<<gb, 256, 0, st>>>(cols->positions, cols->region_of, job->contig_of_region, job->window, flags.as<uint8_t>(), n,
                                        key.as<int64_t>(), idx.as<int64_t>());
        size_t tb = 0;
        PB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, key.as<int64_t>(), key2.as<int64_t>(), idx.as<int64_t>(), order.as<int64_t>(),
                                                (int) n, 0, 64, st));
        PB_TRY(tmp.reserve(tb));
        PB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, key.as<int64_t>(), key2.as<int64_t>(), idx.as<int64_t>(), order.as<int64_t>(),
                                                (int) n, 0, 64, st));
        PB_TRY(head.reserve(4 * n)); PB_TRY(rank.reserve(8 * (n + 1))); PB_TRY(start.reserve(8 * (n + 1)));
        k_site_heads<<<gb, 256, 0, st>>>(key2.as<int64_t>(), n, head.as<int32_t>());
        k_scan_excl<<<1, 1024, 0, st>>>(head.as<int32_t>(), rank.as<int64_t>(), n, nullptr);
        k_site_starts<<<gb, 256, 0, st>>>(head.as<int32_t>(), rank.as<int64_t>(), n, start.as<int64_t>());
        int64_t n_sites = 0;
        PB_CUDA(cudaMemcpyAsync(&n_sites, rank.as<int64_t>() + n, 8, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        VcfArgs A{cols->positions, cols->region_of, cols->depths, cols->freqs, cols->keys, d_probs, flags.as<uint8_t>(), geno.as<uint8_t>(),
                  d_regions, d_ref, job->contig_of_region, job->names, job->name_off, job->vaf_table, order.as<int64_t>(),
                  start.as<int64_t>(), n_sites, *vcf_opt};
        PB_TRY(len.reserve(4 * n_sites)); PB_TRY(has.reserve(4 * n_sites));
        PB_TRY(off.reserve(8 * (n_sites + 1))); PB_TRY(line_of.reserve(8 * (n_sites + 1)));
        const unsigned gs = (unsigned) ceil_div(n_sites, 128);
        k_site_sizes<<<gs, 128, 0, st>>>(A, len.as<int32_t>(), has.as<int32_t>());
        k_scan_excl<<<1, 1024, 0, st>>>(len.as<int32_t>(), off.as<int64_t>(), n_sites, nullptr);
        k_scan_excl<<<1, 1024, 0, st>>>(has.as<int32_t>(), line_of.as<int64_t>(), n_sites, nullptr);
        PB_CUDA(cudaGetLastError());
        PB_CUDA(cudaMemcpyAsync(n_text, off.as<int64_t>() + n_sites, 8, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(n_lines, line_of.as<int64_t>() + n_sites, 8, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        if (!d_text || !d_lines || *n_text > text_cap || *n_lines > lines_cap) {
            set_error("VCF text needs %lld bytes / %lld lines", (long long) *n_text, (long long) *n_lines);
            return PB_ERR_CAPACITY;
        }
        k_site_write<<<gs, 128, 0, st>>>(A, off.as<int64_t>(), line_of.as<int64_t>(), d_text, d_lines);
        PB_CUDA(cudaGetLastError());
        PB_CUDA(cudaStreamSynchronize(st));
        return PB_OK;
    };
    rc = run();
    DevBuf *bufs[] = {&flags, &geno, &key, &key2, &idx, &order, &head, &rank, &start, &len, &has, &off, &line_of, &tmp};
    for (auto *b : bufs) b->release();
    return rc;
}

extern "C" int pb_variant_vcf_host(const int64_t *h_positions, const int32_t *h_region_of, const uint8_t *h_depths, const uint8_t *h_freqs,
                                   const char *h_keys, const float *h_probs, int64_t n, const pb_region_t *h_regions, int64_t n_regions,
                                   const char *h_ref, int64_t ref_bytes, const int32_t *h_contig_of_region, const char *h_names,
                                   const int64_t *h_name_off, int64_t n_contigs, const char *h_vaf_table,
                                   const pb_candidate_options_t *sel_opt, const pb_vcf_options_t *vcf_opt, char *h_text, int64_t text_cap,
                                   pb_vcf_line_t *h_lines, int64_t lines_cap, int64_t *n_text, int64_t *n_lines, void *stream_) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) { set_error("no CUDA device: libpepper_b200 has no CPU fallback"); return PB_ERR_CUDA; }
    if (!n_text || !n_lines || n_contigs < 1 || !h_name_off) { set_error("null argument"); return PB_ERR_ARG; }
    *n_text = 0; *n_lines = 0;
    if (n <= 0) return PB_OK;
    for (int64_t r = 0; r < n_regions; r++)
        if (h_contig_of_region[r] < 0 || h_contig_of_region[r] >= n_contigs) { set_error("contig_of_region[%lld] out of range", (long long) r); return PB_ERR_ARG; }
    for (int64_t i = 0; i < n; i++)
        if (h_region_of[i] < 0 || h_region_of[i] >= n_regions) { set_error("region_of[%lld] out of range", (long long) i); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    DevBuf p, r, d, f, k, pr, rg, rf, cr, nm, no, vt, tx, ln;
    auto run = [&]() -> int {
        PB_TRY(upload(p, h_positions, sizeof(int64_t) * n, st));
        PB_TRY(upload(r, h_region_of, sizeof(int32_t) * n, st));
        PB_TRY(upload(d, h_depths, n, st));
        PB_TRY(upload(f, h_freqs, n, st));
        PB_TRY(upload(k, h_keys, (size_t) n * PB_ALLELE_STRIDE, st));
        PB_TRY(upload(pr, h_probs, sizeof(float) * 3 * n, st));
        PB_TRY(upload(rg, h_regions, sizeof(pb_region_t) * n_regions, st));
        PB_TRY(upload(rf, h_ref, (size_t) ref_bytes, st));
        PB_TRY(upload(cr, h_contig_of_region, sizeof(int32_t) * n_regions, st));
        PB_TRY(nm.reserve((size_t) h_name_off[n_contigs] + 1));
        if (h_name_off[n_contigs] > 0) PB_TRY(upload(nm, h_names, (size_t) h_name_off[n_contigs], st));
        PB_TRY(upload(no, h_name_off, sizeof(int64_t) * (n_contigs + 1), st));
        PB_TRY(upload(vt, h_vaf_table, 256 * 256 * VAF_STRIDE, st));
        PB_TRY(tx.reserve(text_cap > 0 ? text_cap : 1)); PB_TRY(ln.reserve(sizeof(pb_vcf_line_t) * (lines_cap > 0 ? lines_cap : 1)));
        pb_candidate_columns_t cols{p.as<int64_t>(), r.as<int32_t>(), d.as<uint8_t>(), f.as<uint8_t>(), k.as<char>()};
        pb_vcf_job_t job{cr.as<int32_t>(), nm.as<char>(), no.as<int64_t>(), vt.as<char>(), nullptr};
        PB_TRY(pb_variant_vcf_device(&cols, pr.as<float>(), n, rg.as<pb_region_t>(), rf.as<char>(), &job, sel_opt, vcf_opt,
                                     h_text ? tx.as<char>() : nullptr, text_cap, h_lines ? ln.as<pb_vcf_line_t>() : nullptr, lines_cap,
                                     n_text, n_lines, stream_));
        PB_CUDA(cudaMemcpyAsync(h_text, tx.p, (size_t) *n_text, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_lines, ln.p, sizeof(pb_vcf_line_t) * *n_lines, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        return PB_OK;
    };
    const int rc = run();
    DevBuf *bufs[] = {&p, &r, &d, &f, &k, &pr, &rg, &rf, &cr, &nm, &no, &vt, &tx, &ln};
    for (auto *b : bufs) b->release();
    return rc;
}

extern "C" int pb_vcf_gather_lines_device(const char *d_text, const pb_vcf_line_t *d_lines, const int64_t *d_sel, const int64_t *d_dst,
                                          int64_t n, uint8_t *d_out, void *stream_) {
    if (n <= 0) return PB_OK;
    if (!d_text || !d_lines || !d_sel || !d_dst || !d_out) { set_error("null argument"); return PB_ERR_ARG; }
    k_gather_lines<<<(unsigned) ceil_div(n * 32, 256), 256, 0, (cudaStream_t) stream_>>>(d_text, d_lines, d_sel, d_dst, n, d_out);
    PB_CUDA(cudaGetLastError());
    return PB_OK;
}

extern "C" int pb_test_format_g(const float *h_x, int64_t n, char *h_out) {
    if (n <= 0) return PB_OK;
    if (!h_x || !h_out) { set_error("null argument"); return PB_ERR_ARG; }
    DevBuf x, o;
    auto run = [&]() -> int {
        PB_TRY(upload(x, h_x, sizeof(float) * n, 0));
        PB_TRY(o.reserve((size_t) n * 16));
        k_format_g<<<(unsigned) ceil_div(n, 256), 256>>>(x.as<float>(), n, o.as<char>());
        PB_CUDA(cudaGetLastError());
        PB_CUDA(cudaMemcpy(h_out, o.p, (size_t) n * 16, cudaMemcpyDeviceToHost));
        return PB_OK;
    };
    const int rc = run();
    x.release(); o.release();
    return rc;
}

extern "C" int pb_test_vcf_qual(const float *h_p, int64_t n, int32_t *h_qual) {
    if (n <= 0) return PB_OK;
    if (!h_p || !h_qual) { set_error("null argument"); return PB_ERR_ARG; }
    DevBuf p, q;
    auto run = [&]() -> int {
        PB_TRY(upload(p, h_p, sizeof(float) * n, 0));
        PB_TRY(q.reserve(sizeof(int32_t) * n));
        k_vcf_qual<<<(unsigned) ceil_div(n, 256), 256>>>(p.as<float>(), n, q.as<int32_t>());
        PB_CUDA(cudaGetLastError());
        PB_CUDA(cudaMemcpy(h_qual, q.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
        return PB_OK;
    };
    const int rc = run();
    p.release(); q.release();
    return rc;
}
