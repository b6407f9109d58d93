// gVCF reference blocks on the device (DESIGN.md section 4, "gVCF"): from the encoder's track of (n_ref, n_alt) pairs, the
// segments of the owned windows and the masked ranges of the written records, the block lines of PEPPER_VARIANT.g.vcf.gz; and
// the record lines, PEPPER_VARIANT_FULL's lines with the <*> allele.
//
//   k_gvcf_mask      per masked range: the positions no block may take
//   k_gvcf_breaks    per segment: its first position (a block never crosses it)
//   k_gvcf_runs      per tile of GV_TILE positions: block starts and ends (count pass), then, after two scans, both in order
//   k_gvcf_block     one warp per block: the first position of least GQ and the least DP
//   k_gvcf_format    one thread per block: the line's length (count pass) or text (write pass), after one scan
//   k_gvcf_records   one thread per record line: the FULL line with ",<*>" and ",." inserted
//
// PL and GQ are computed with __dmul_rn / __dadd_rn / __dsub_rn only (no contraction), so each value is the one numpy's float64
// arithmetic gives for the same expression.
#include "handles.cuh"
#include <cub/block/block_scan.cuh>
#include <algorithm>

namespace pb {

constexpr int GV_THREADS = 256, GV_PER = 8, GV_TILE = GV_THREADS * GV_PER;
constexpr int GV_MASKED = -2;

struct GvcfModel { double a, b, h; int binsize; };

// PL of 0/0, 0/1, 1/1 and GQ of one track value; returns DP
__device__ __forceinline__ int gv_likelihoods(uint32_t v, const GvcfModel &M, int64_t pl[3], int &gq) {
    const int nr = (int) (v & 0xffffu), na = (int) (v >> 16);
    const double r = (double) nr, x = (double) na;
    const double l00 = __dadd_rn(__dmul_rn(r, M.a), __dmul_rn(x, M.b));
    const double l01 = __dmul_rn(__dadd_rn(r, x), M.h);
    const double l11 = __dadd_rn(__dmul_rn(r, M.b), __dmul_rn(x, M.a));
    const double mx = fmax(l00, fmax(l01, l11));
    const double l[3] = {l00, l01, l11};
#pragma unroll
    for (int g = 0; g < 3; g++) pl[g] = (int64_t) floor(__dadd_rn(__dmul_rn(10.0, __dsub_rn(mx, l[g])), 0.5));
    gq = (int) min((int64_t) 99, max((int64_t) 0, min(pl[1], pl[2]) - pl[0]));
    return nr + na;
}

__device__ __forceinline__ int gv_key(const uint32_t *track, const uint8_t *mask, int64_t t, const GvcfModel &M) {
    if (mask[t]) return GV_MASKED;
    int64_t pl[3];
    int gq;
    const int dp = gv_likelihoods(track[t], M, pl, gq);
    return dp == 0 ? -1 : gq / M.binsize;
}

__global__ void k_gvcf_mask(const int64_t *__restrict__ ranges, int64_t T, uint8_t *__restrict__ mask) {
    const int64_t a = max(ranges[2 * blockIdx.x], (int64_t) 0), b = min(ranges[2 * blockIdx.x + 1], T);
    for (int64_t t = a + threadIdx.x; t < b; t += blockDim.x) mask[t] = 1;
}

__global__ void k_gvcf_breaks(const pb_gvcf_segment_t *__restrict__ seg, int64_t n, uint8_t *__restrict__ brk) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && seg[i].len > 0) brk[seg[i].toff] = 1;
}

// block starts / ends of each tile; WRITE: their track indices in order from the scanned slots
template <bool WRITE>
__global__ void __launch_bounds__(GV_THREADS) k_gvcf_runs(const uint32_t *__restrict__ track, const uint8_t *__restrict__ mask,
                                                          const uint8_t *__restrict__ brk, int64_t T, GvcfModel M,
                                                          int32_t *__restrict__ n_start, int32_t *__restrict__ n_end,
                                                          const int64_t *__restrict__ o_start, const int64_t *__restrict__ o_end,
                                                          int64_t *__restrict__ ra, int64_t *__restrict__ rb) {
    using Scan = cub::BlockScan<int, GV_THREADS>;
    __shared__ typename Scan::TempStorage tmp[2];
    const int64_t p0 = (int64_t) blockIdx.x * GV_TILE + (int64_t) threadIdx.x * GV_PER;
    int key[GV_PER + 2];                      // keys of p0 - 1 .. p0 + GV_PER
#pragma unroll
    for (int k = 0; k < GV_PER + 2; k++) {
        const int64_t t = p0 - 1 + k;
        key[k] = (t >= 0 && t < T) ? gv_key(track, mask, t, M) : GV_MASKED;
    }
    unsigned fs = 0, fe = 0;
#pragma unroll
    for (int k = 0; k < GV_PER; k++) {
        const int64_t t = p0 + k;
        if (t < T && key[k + 1] != GV_MASKED) {
            if (brk[t] || key[k] != key[k + 1]) fs |= 1u << k;
            if (t + 1 == T || brk[t + 1] || key[k + 2] != key[k + 1]) fe |= 1u << k;
        }
    }
    int xs, xe, ts, te;
    Scan(tmp[0]).ExclusiveSum(__popc(fs), xs, ts);
    Scan(tmp[1]).ExclusiveSum(__popc(fe), xe, te);
    if (!WRITE) {
        if (threadIdx.x == 0) { n_start[blockIdx.x] = ts; n_end[blockIdx.x] = te; }
        return;
    }
    int64_t os = o_start[blockIdx.x] + xs, oe = o_end[blockIdx.x] + xe;
    for (int k = 0; k < GV_PER; k++) {
        if (fs >> k & 1u) ra[os++] = p0 + k;
        if (fe >> k & 1u) rb[oe++] = p0 + k;
    }
}

// one warp per block [ra, rb]: info[3k] = least GQ, [3k + 1] = least DP, [3k + 2] = first track index of least GQ
__global__ void k_gvcf_block(const uint32_t *__restrict__ track, const int64_t *__restrict__ ra, const int64_t *__restrict__ rb,
                             int64_t n_blocks, GvcfModel M, int64_t *__restrict__ info) {
    const int64_t k = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (k >= n_blocks) return;
    const int64_t a = ra[k], b = rb[k];
    int best_gq = INT_MAX, best_dp = INT_MAX;
    int64_t best_t = INT64_MAX;
    for (int64_t t = a + lane; t <= b; t += 32) {
        int64_t pl[3];
        int gq;
        const int dp = gv_likelihoods(track[t], M, pl, gq);
        if (gq < best_gq) { best_gq = gq; best_t = t; }          // t ascends per lane: the first of this lane's least
        best_dp = min(best_dp, dp);
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        const int og = __shfl_xor_sync(0xffffffffu, best_gq, d), od = __shfl_xor_sync(0xffffffffu, best_dp, d);
        const int64_t ot = __shfl_xor_sync(0xffffffffu, best_t, d);
        if (og < best_gq || (og == best_gq && ot < best_t)) { best_gq = og; best_t = ot; }
        best_dp = min(best_dp, od);
    }
    if (lane == 0) { info[3 * k] = best_gq; info[3 * k + 1] = best_dp; info[3 * k + 2] = best_t; }
}

__device__ __forceinline__ int gv_int(char *out, int64_t v) {      // v >= 0
    char t[20];
    int n = 0;
    do { t[n++] = (char) ('0' + v % 10); v /= 10; } while (v);
    if (out) for (int i = 0; i < n; i++) out[i] = t[n - 1 - i];
    return n;
}

struct GvcfView {
    const uint32_t *track;
    const pb_gvcf_segment_t *seg; int64_t n_seg;
    const char *ref, *names; const int64_t *name_off;
    GvcfModel M;
};

// WRITE: the text at text_off[k], the line's row in lines[k]; otherwise its bytes to tlen[k]
template <bool WRITE>
__global__ void k_gvcf_format(GvcfView V, const int64_t *__restrict__ ra, const int64_t *__restrict__ rb,
                              const int64_t *__restrict__ info, int64_t n_blocks, int32_t *__restrict__ tlen,
                              const int64_t *__restrict__ text_off, char *__restrict__ text, pb_vcf_line_t *__restrict__ lines) {
    const int64_t k = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_blocks) return;
    const int64_t a = ra[k], b = rb[k];
    int64_t lo = 0, hi = V.n_seg - 1;                  // the last segment starting at or before a
    while (lo < hi) {
        const int64_t m = (lo + hi + 1) >> 1;
        if (V.seg[m].toff <= a) lo = m; else hi = m - 1;
    }
    const pb_gvcf_segment_t s = V.seg[lo];
    const int64_t pos = s.pos0 + (a - s.toff), last1 = s.pos0 + (b - s.toff) + 1;
    char r = to_upper(V.ref[s.ref_off + (a - s.toff)]);
    if (!is_upper_acgt(r)) r = 'N';
    const int64_t gq = info[3 * k], dp = info[3 * k + 1];
    int64_t pl[3];
    int gq2;
    gv_likelihoods(V.track[info[3 * k + 2]], V.M, pl, gq2);
    const bool nocall = dp == 0;
    const int64_t n0 = V.name_off[s.contig], nlen = V.name_off[s.contig + 1] - n0;
    // CHROM POS . REF <*> . . END=x GT:GQ:MIN_DP:PL 0/0:gq:dp:pl0,pl1,pl2
    const int64_t n = nlen + 1 + gv_int(nullptr, pos + 1) + 3 + 1 + 1 + 3 + 4 + 5 + gv_int(nullptr, last1) + 1 + 15 + 1 + 3 + 1 +
                      gv_int(nullptr, gq) + 1 + gv_int(nullptr, dp) + 1 + gv_int(nullptr, pl[0]) + 1 + gv_int(nullptr, pl[1]) + 1 +
                      gv_int(nullptr, pl[2]) + 1;
    if (!WRITE) { tlen[k] = (int32_t) n; return; }
    char *o = text + text_off[k];
    for (int64_t i = 0; i < nlen; i++) *o++ = V.names[n0 + i];
    *o++ = '\t';
    o += gv_int(o, pos + 1);
    *o++ = '\t'; *o++ = '.'; *o++ = '\t'; *o++ = r; *o++ = '\t';
    const char *alt = "<*>\t.\t.\tEND=";
    for (int i = 0; i < 12; i++) *o++ = alt[i];
    o += gv_int(o, last1);
    const char *fmt = "\tGT:GQ:MIN_DP:PL\t";
    for (int i = 0; i < 17; i++) *o++ = fmt[i];
    *o++ = nocall ? '.' : '0'; *o++ = '/'; *o++ = nocall ? '.' : '0'; *o++ = ':';
    o += gv_int(o, gq); *o++ = ':';
    o += gv_int(o, dp); *o++ = ':';
    o += gv_int(o, pl[0]); *o++ = ',';
    o += gv_int(o, pl[1]); *o++ = ',';
    o += gv_int(o, pl[2]); *o++ = '\n';
    pb_vcf_line_t L;
    L.pos = pos; L.text_off = text_off[k]; L.contig = s.contig; L.ref_len = (int32_t) (b - a + 1); L.cls = PB_GVCF_CLASS_BLOCK;
    L.text_len = (int32_t) n;
    lines[k] = L;
}

// FORMAT GT:AP:GQ:DP:AD:VAF:REP: the Number=A values end before the sample column's 2nd, 5th and 6th ':'
__global__ void k_gvcf_records(const char *__restrict__ text, const pb_vcf_line_t *__restrict__ lines, int64_t n,
                               const int64_t *__restrict__ out_off, char *__restrict__ out) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const pb_vcf_line_t L = lines[i];
    const char *src = text + L.text_off;
    char *o = out + out_off[i];
    int tabs = 0, colons = 0;
    for (int j = 0; j < L.text_len; j++) {
        const char c = src[j];
        if (c == '\t') {
            if (tabs == 4) { *o++ = ','; *o++ = '<'; *o++ = '*'; *o++ = '>'; }
            tabs++;
        } else if (tabs == 9 && (c == ':' || c == '\n')) {
            colons++;
            if (colons == 2 || colons == 5 || colons == 6) { *o++ = ','; *o++ = '.'; }
        }
        *o++ = c;
    }
}

}  // namespace pb

using namespace pb;

extern "C" int pb_gvcf_blocks_device(const uint32_t *d_track, int64_t n_track, const pb_gvcf_segment_t *h_segments, int64_t n_segments,
                                     const int64_t *h_masks, int64_t n_masks, const char *d_ref, const char *h_names,
                                     const int64_t *h_name_off, int64_t n_contigs, const pb_gvcf_params_t *params, char *d_text,
                                     int64_t text_cap, pb_vcf_line_t *d_lines, int64_t lines_cap, int64_t *n_text, int64_t *n_lines,
                                     void *stream_) {
    if (!n_text || !n_lines || !params || params->binsize <= 0 || n_track < 0 || (n_track > 0 && (!d_track || !d_ref)) ||
        (n_segments > 0 && !h_segments) || (n_masks > 0 && !h_masks) || !h_names || !h_name_off || n_contigs < 0) {
        set_error("bad argument"); return PB_ERR_ARG;
    }
    *n_text = 0; *n_lines = 0;
    if (n_track == 0) return PB_OK;
    int64_t covered = 0;
    for (int64_t i = 0; i < n_segments; i++) {
        const pb_gvcf_segment_t &s = h_segments[i];
        if (s.toff != covered || s.len < 0 || s.contig < 0 || s.contig >= n_contigs) {
            set_error("segment %lld: segments must tile the track in order with valid contigs", (long long) i); return PB_ERR_ARG;
        }
        covered += s.len;
    }
    if (covered != n_track) { set_error("segments cover %lld of %lld track positions", (long long) covered, (long long) n_track); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    const GvcfModel M{params->a, params->b, params->h, params->binsize};
    const int64_t tiles = (n_track + GV_TILE - 1) / GV_TILE;
    DevBuf mask, brk, seg, rng, cnt[2], off[2], ra, rb, info, tlen, toff, names, noff;
    int rc = PB_OK;
    do {
        if ((rc = mask.reserve((size_t) n_track)) != PB_OK || (rc = brk.reserve((size_t) n_track)) != PB_OK) break;
        if (cudaMemsetAsync(mask.p, 0, (size_t) n_track, st) != cudaSuccess || cudaMemsetAsync(brk.p, 0, (size_t) n_track, st) != cudaSuccess) {
            set_error("memset failed"); rc = PB_ERR_CUDA; break;
        }
        if ((rc = upload(seg, h_segments, sizeof(pb_gvcf_segment_t) * n_segments, st)) != PB_OK) break;
        if ((rc = upload(names, h_names, (size_t) h_name_off[n_contigs], st)) != PB_OK) break;
        if ((rc = upload(noff, h_name_off, sizeof(int64_t) * (n_contigs + 1), st)) != PB_OK) break;
        if (n_masks > 0) {
            if ((rc = upload(rng, h_masks, sizeof(int64_t) * 2 * n_masks, st)) != PB_OK) break;
            k_gvcf_mask<<<(unsigned) n_masks, 256, 0, st>>>(rng.as<int64_t>(), n_track, mask.as<uint8_t>());
        }
        if (n_segments > 0)
            k_gvcf_breaks<<<(unsigned) ((n_segments + 255) / 256), 256, 0, st>>>(seg.as<pb_gvcf_segment_t>(), n_segments, brk.as<uint8_t>());
        for (int i = 0; i < 2 && rc == PB_OK; i++) {
            rc = cnt[i].reserve(sizeof(int32_t) * tiles);
            if (rc == PB_OK) rc = off[i].reserve(sizeof(int64_t) * (tiles + 1));
        }
        if (rc != PB_OK) break;
        k_gvcf_runs<false><<<(unsigned) tiles, GV_THREADS, 0, st>>>(d_track, mask.as<uint8_t>(), brk.as<uint8_t>(), n_track, M,
                                                                    cnt[0].as<int32_t>(), cnt[1].as<int32_t>(), nullptr, nullptr, nullptr, nullptr);
        for (int i = 0; i < 2; i++) k_scan_excl<<<1, 1024, 0, st>>>(cnt[i].as<int32_t>(), off[i].as<int64_t>(), tiles, nullptr);
        int64_t nb = 0;
        PB_CUDA(cudaMemcpyAsync(&nb, off[0].as<int64_t>() + tiles, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        *n_lines = nb;
        if (nb == 0) break;
        if ((rc = ra.reserve(sizeof(int64_t) * nb)) != PB_OK || (rc = rb.reserve(sizeof(int64_t) * nb)) != PB_OK) break;
        if ((rc = info.reserve(sizeof(int64_t) * 3 * nb)) != PB_OK || (rc = tlen.reserve(sizeof(int32_t) * nb)) != PB_OK) break;
        if ((rc = toff.reserve(sizeof(int64_t) * (nb + 1))) != PB_OK) break;
        k_gvcf_runs<true><<<(unsigned) tiles, GV_THREADS, 0, st>>>(d_track, mask.as<uint8_t>(), brk.as<uint8_t>(), n_track, M, nullptr,
                                                                   nullptr, off[0].as<int64_t>(), off[1].as<int64_t>(), ra.as<int64_t>(),
                                                                   rb.as<int64_t>());
        k_gvcf_block<<<(unsigned) ((nb + 7) / 8), 256, 0, st>>>(d_track, ra.as<int64_t>(), rb.as<int64_t>(), nb, M, info.as<int64_t>());
        GvcfView V{d_track, seg.as<pb_gvcf_segment_t>(), n_segments, d_ref, names.as<char>(), noff.as<int64_t>(), M};
        const unsigned g = (unsigned) ((nb + 127) / 128);
        k_gvcf_format<false><<<g, 128, 0, st>>>(V, ra.as<int64_t>(), rb.as<int64_t>(), info.as<int64_t>(), nb, tlen.as<int32_t>(),
                                                nullptr, nullptr, nullptr);
        k_scan_excl<<<1, 1024, 0, st>>>(tlen.as<int32_t>(), toff.as<int64_t>(), nb, nullptr);
        PB_CUDA(cudaMemcpyAsync(n_text, toff.as<int64_t>() + nb, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        if (!d_text || !d_lines || nb > lines_cap || *n_text > text_cap) {
            set_error("gVCF capacity (%lld lines, %lld bytes) < (%lld, %lld) needed", (long long) lines_cap, (long long) text_cap,
                      (long long) nb, (long long) *n_text);
            rc = PB_ERR_CAPACITY; break;
        }
        k_gvcf_format<true><<<g, 128, 0, st>>>(V, ra.as<int64_t>(), rb.as<int64_t>(), info.as<int64_t>(), nb, nullptr,
                                               toff.as<int64_t>(), d_text, d_lines);
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("gVCF blocks: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    } while (0);
    if (rc == PB_OK) {
        cudaError_t e = cudaStreamSynchronize(st);
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e != cudaSuccess) { set_error("gVCF blocks: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    } else {
        cudaStreamSynchronize(st);
    }
    DevBuf *bufs[] = {&mask, &brk, &seg, &rng, &cnt[0], &cnt[1], &off[0], &off[1], &ra, &rb, &info, &tlen, &toff, &names, &noff};
    for (auto *x : bufs) x->release();
    return rc;
}

extern "C" int pb_gvcf_blocks_host(const uint32_t *h_track, int64_t n_track, const pb_gvcf_segment_t *h_segments, int64_t n_segments,
                                   const int64_t *h_masks, int64_t n_masks, const char *h_ref, int64_t ref_bytes, const char *h_names,
                                   const int64_t *h_name_off, int64_t n_contigs, const pb_gvcf_params_t *params, char *h_text,
                                   int64_t text_cap, pb_vcf_line_t *h_lines, int64_t lines_cap, int64_t *n_text, int64_t *n_lines,
                                   void *stream_) {
    if (!n_text || !n_lines || (n_track > 0 && (!h_track || !h_ref))) { set_error("bad argument"); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    DevBuf track, ref, text, lines;
    int rc = PB_OK;
    do {
        if ((rc = upload(track, h_track, sizeof(uint32_t) * std::max<int64_t>(n_track, 0), st)) != PB_OK) break;
        if ((rc = upload(ref, h_ref, (size_t) std::max<int64_t>(ref_bytes, 0), st)) != PB_OK) break;
        if ((rc = text.reserve((size_t) std::max<int64_t>(text_cap, 1))) != PB_OK) break;
        if ((rc = lines.reserve(sizeof(pb_vcf_line_t) * std::max<int64_t>(lines_cap, 1))) != PB_OK) break;
        rc = pb_gvcf_blocks_device(track.as<uint32_t>(), n_track, h_segments, n_segments, h_masks, n_masks, ref.as<char>(), h_names,
                                   h_name_off, n_contigs, params, h_text ? text.as<char>() : nullptr, text_cap,
                                   h_lines ? lines.as<pb_vcf_line_t>() : nullptr, lines_cap, n_text, n_lines, stream_);
        if (rc != PB_OK) break;
        if (*n_text > 0 && cudaMemcpyAsync(h_text, text.p, (size_t) *n_text, cudaMemcpyDeviceToHost, st) != cudaSuccess) { rc = PB_ERR_CUDA; break; }
        if (*n_lines > 0 && cudaMemcpyAsync(h_lines, lines.p, sizeof(pb_vcf_line_t) * *n_lines, cudaMemcpyDeviceToHost, st) != cudaSuccess) {
            rc = PB_ERR_CUDA; break;
        }
        if (cudaStreamSynchronize(st) != cudaSuccess) { set_error("gVCF blocks: copy failed"); rc = PB_ERR_CUDA; }
    } while (0);
    DevBuf *bufs[] = {&track, &ref, &text, &lines};
    for (auto *x : bufs) x->release();
    return rc;
}

extern "C" int pb_gvcf_records_device(const char *d_text, const pb_vcf_line_t *d_lines, int64_t n, const int64_t *d_out_off, char *d_out,
                                      void *stream_) {
    if (n < 0 || (n > 0 && (!d_text || !d_lines || !d_out_off || !d_out))) { set_error("bad argument"); return PB_ERR_ARG; }
    if (n == 0) return PB_OK;
    k_gvcf_records<<<(unsigned) ((n + 127) / 128), 128, 0, (cudaStream_t) stream_>>>(d_text, d_lines, n, d_out_off, d_out);
    PB_CUDA(cudaGetLastError());
    return PB_OK;
}
