// The edits VCF of a polished contig on the device: from the edit events of an edits session (stitch.cu edit_columns) and the
// draft, the records that turn upper(draft[span]) into the polished sequence (DESIGN.md section 4, "Polish edits").
//
//   k_edit_cover     per coverage range: the positions an image won at index 0
//   k_edit_marks     per event: the positions with an index-0 event or an insertion after them; a position is edited when it
//                    has either or no image won it
//   k_runs           per tile of positions: run starts and ends (count pass), then, after two scans, both in order (the k-th
//                    start and the k-th end bound run k)
//   k_run_info       one thread per run: its ALT length
//   k_run_format     one thread per run: the record's line length (count pass) or text (write pass), after one scan
#include "handles.cuh"
#include <cub/block/block_scan.cuh>
#include <algorithm>
#include <cstring>

namespace pb {

constexpr int ED_THREADS = 256, ED_PER = 8, ED_TILE = ED_THREADS * ED_PER;
constexpr uint8_t ED_NONE = 255;            // QUAL of a run without an event: '.'

// mark bits: 1 = an index-0 event (deletion or substitution), 2 = an insertion after the position, 4 = won by an image
__global__ void k_edit_marks(const pb_edit_event_t *__restrict__ ev, int64_t n, int64_t s0, int64_t L, uint8_t *__restrict__ mark) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t p = ev[i].position - s0;
    if (p < 0 || p >= L) return;
    const unsigned bit = ev[i].index == 0 ? 1u : 2u;
    // byte-wise OR through the aligned word (an index-0 event and the insertions after it share the byte)
    unsigned *w = reinterpret_cast<unsigned *>(reinterpret_cast<uintptr_t>(mark + p) & ~(uintptr_t) 3);
    atomicOr(w, bit << (8 * (reinterpret_cast<uintptr_t>(mark + p) & 3)));
}

// one block per coverage range [first, last] (a range is at most one image wide)
__global__ void k_edit_cover(const int64_t *__restrict__ cover, int64_t s0, int64_t L, uint8_t *__restrict__ mark) {
    const int64_t a = std::max<int64_t>(cover[2 * blockIdx.x] - s0, 0), b = std::min<int64_t>(cover[2 * blockIdx.x + 1] - s0, L - 1);
    for (int64_t p = a + threadIdx.x; p <= b; p += blockDim.x) {
        unsigned *w = reinterpret_cast<unsigned *>(reinterpret_cast<uintptr_t>(mark + p) & ~(uintptr_t) 3);
        atomicOr(w, 4u << (8 * (reinterpret_cast<uintptr_t>(mark + p) & 3)));
    }
}

__device__ __forceinline__ bool edited(const uint8_t *mark, int64_t p) { return mark[p] != 4; }

// run starts / ends of each tile of ED_TILE positions; WRITE: their span offsets in order from the scanned slots
template <bool WRITE>
__global__ void __launch_bounds__(ED_THREADS) k_runs(const uint8_t *__restrict__ mark, int64_t L, int32_t *__restrict__ n_start,
                                                     int32_t *__restrict__ n_end, const int64_t *__restrict__ o_start,
                                                     const int64_t *__restrict__ o_end, int64_t *__restrict__ ra, int64_t *__restrict__ rb) {
    using Scan = cub::BlockScan<int, ED_THREADS>;
    __shared__ typename Scan::TempStorage tmp[2];
    const int64_t p0 = (int64_t) blockIdx.x * ED_TILE + (int64_t) threadIdx.x * ED_PER;
    unsigned fs = 0, fe = 0;
#pragma unroll
    for (int k = 0; k < ED_PER; k++) {
        const int64_t p = p0 + k;
        if (p < L && edited(mark, p)) {
            if (p == 0 || !edited(mark, p - 1)) fs |= 1u << k;
            if (p == L - 1 || !edited(mark, p + 1)) fe |= 1u << k;
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
    for (int k = 0; k < ED_PER; k++) {
        if (fs >> k & 1u) ra[os++] = p0 + k;
        if (fe >> k & 1u) rb[oe++] = p0 + k;
    }
}

// first event at or after draft position q (events sorted by (position, index))
__device__ int64_t lower_event(const pb_edit_event_t *ev, int64_t n, int64_t q) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t m = (lo + hi) >> 1;
        if (ev[m].position < q) lo = m + 1; else hi = m;
    }
    return lo;
}

struct EditView {
    const pb_edit_event_t *ev; int64_t n_ev;
    const uint8_t *mark; const char *draft; int64_t s0, L;
};

__device__ __forceinline__ char upper(char c) { return (c >= 'a' && c <= 'z') ? (char) (c - 32) : c; }

// ALT of draft positions [a, b] (span offsets): per position the winner's base (the draft base when it is an identity; nothing
// when it is deleted or uncovered) and then its inserted bases.  Writes to `out` when set; returns the length, and the least
// phred and whether a position is uncovered
__device__ int64_t alt_walk(const EditView &V, int64_t a, int64_t b, char *out, int *qual, bool *uncov) {
    int64_t j = lower_event(V.ev, V.n_ev, V.s0 + a), len = 0;
    int q = ED_NONE;
    bool u = false;
    for (int64_t p = a; p <= b; p++) {
        const int64_t pos = V.s0 + p;
        if (j < V.n_ev && V.ev[j].position == pos && V.ev[j].index == 0) {
            q = min(q, (int) V.ev[j].phred);
            if (V.ev[j].label) { if (out) out[len] = "ACGT"[V.ev[j].label - 1]; len++; }
            j++;
        } else if (!(V.mark[p] & 4)) {
            u = true;
        } else {
            if (out) out[len] = upper(V.draft[p]);
            len++;
        }
        for (; j < V.n_ev && V.ev[j].position == pos; j++) {
            q = min(q, (int) V.ev[j].phred);
            if (out) out[len] = "ACGT"[V.ev[j].label - 1];
            len++;
        }
    }
    *qual = q; *uncov = u;
    return len;
}

__global__ void k_run_info(EditView V, const int64_t *__restrict__ ra, const int64_t *__restrict__ rb, int64_t n_runs,
                           int64_t *__restrict__ alt_len) {
    const int64_t k = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_runs) return;
    int q; bool u;
    alt_len[k] = alt_walk(V, ra[k], rb[k], nullptr, &q, &u);
}

__device__ int write_int(char *out, int64_t v) {
    char t[20];
    int n = 0;
    do { t[n++] = (char) ('0' + v % 10); v /= 10; } while (v);
    if (out) for (int i = 0; i < n; i++) out[i] = t[n - 1 - i];
    return n;
}

// One record per run.  A run whose ALT is empty takes the identity base before it, or at the span's first base the one after
// it; when that base is also the left anchor of the next run (which then starts two after this one, with an empty ALT), the
// two runs are one record over both and the base between them.  WRITE: the text at text_off[k] and (0-based POS, REF length,
// text bytes) to lines[k]; otherwise the text bytes to tlen[k] (0: the run is part of the record before it).
template <bool WRITE>
__global__ void k_run_format(EditView V, const int64_t *__restrict__ ra, const int64_t *__restrict__ rb, const int64_t *__restrict__ alt_len,
                             int64_t n_runs, const char *__restrict__ name, int name_len, int32_t *__restrict__ tlen,
                             const int64_t *__restrict__ text_off, char *__restrict__ text, int64_t *__restrict__ lines) {
    const int64_t k = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_runs) return;
    const bool pair = n_runs > 1 && ra[0] == 0 && alt_len[0] == 0 && alt_len[1] == 0 && ra[1] == rb[0] + 2;
    if (k == 1 && pair) {
        if (!WRITE) tlen[k] = 0;
        else { lines[3 * k] = -1; lines[3 * k + 1] = 0; lines[3 * k + 2] = 0; }
        return;
    }
    const int64_t a = ra[k], b = (k == 0 && pair) ? rb[1] : rb[k];
    int q; bool u;
    const int64_t alen = alt_walk(V, a, b, nullptr, &q, &u);
    // the anchor: -1 before, +1 after, 0 none
    const int anchor = alen > 0 ? 0 : (a > 0 ? -1 : (b + 1 < V.L ? 1 : 0));
    const int64_t r0 = anchor < 0 ? a - 1 : a, r1 = anchor > 0 ? b + 1 : b;
    const int64_t pos1 = V.s0 + r0 + 1;
    int64_t n = name_len + 1 + write_int(nullptr, pos1) + 3 + (r1 - r0 + 1) + 1 + alen + (anchor ? 1 : 0) + 1 +
                (q == ED_NONE ? 1 : write_int(nullptr, q)) + 3 + (u ? 9 : 1) + 1;
    if (!WRITE) { tlen[k] = (int32_t) n; return; }
    char *o = text + text_off[k];
    for (int i = 0; i < name_len; i++) *o++ = name[i];
    *o++ = '\t';
    o += write_int(o, pos1);
    *o++ = '\t'; *o++ = '.'; *o++ = '\t';
    for (int64_t p = r0; p <= r1; p++) *o++ = upper(V.draft[p]);
    *o++ = '\t';
    if (anchor < 0) *o++ = upper(V.draft[a - 1]);
    alt_walk(V, a, b, o, &q, &u);
    o += alen;
    if (anchor > 0) *o++ = upper(V.draft[b + 1]);
    *o++ = '\t';
    if (q == ED_NONE) *o++ = '.'; else o += write_int(o, q);
    *o++ = '\t'; *o++ = '.'; *o++ = '\t';
    if (u) { const char *f = "UNCOVERED"; for (int i = 0; i < 9; i++) *o++ = f[i]; } else *o++ = '.';
    *o++ = '\n';
    lines[3 * k] = V.s0 + r0; lines[3 * k + 1] = r1 - r0 + 1; lines[3 * k + 2] = n;
}

}  // namespace pb

using namespace pb;

extern "C" int pb_polish_edits_vcf_device(const pb_edit_event_t *d_events, int64_t n_events, const int64_t *h_cover, int64_t n_cover,
                                          int64_t span_start, int64_t span_end, const char *d_draft, const char *contig,
                                          char *d_text, int64_t capacity_text, int64_t *d_lines, int64_t capacity_lines,
                                          int64_t *n_lines, int64_t *n_text, void *stream_) {
    if (!n_lines || !n_text || !contig || !d_draft || (n_events > 0 && !d_events) || (n_cover > 0 && !h_cover) || span_end < span_start) {
        set_error("bad argument"); return PB_ERR_ARG;
    }
    cudaStream_t st = (cudaStream_t) stream_;
    *n_lines = 0; *n_text = 0;
    const int64_t L = span_end - span_start + 1, tiles = (L + ED_TILE - 1) / ED_TILE;
    const int name_len = (int) strlen(contig);
    DevBuf mark, cover, cnt[2], off[2], ra, rb, alt, tlen, toff, name;
    int rc = PB_OK;
    do {
        if ((rc = mark.reserve((size_t) L + 4)) != PB_OK) break;
        if (cudaMemsetAsync(mark.p, 0, (size_t) L + 4, st) != cudaSuccess) { set_error("memset failed"); rc = PB_ERR_CUDA; break; }
        if (n_cover > 0) {
            if ((rc = upload(cover, h_cover, sizeof(int64_t) * 2 * n_cover, st)) != PB_OK) break;
            k_edit_cover<<<(unsigned) n_cover, 256, 0, st>>>(cover.as<int64_t>(), span_start, L, mark.as<uint8_t>());
        }
        if (n_events > 0) k_edit_marks<<<(unsigned) ((n_events + 255) / 256), 256, 0, st>>>(d_events, n_events, span_start, L, mark.as<uint8_t>());
        for (int i = 0; i < 2 && rc == PB_OK; i++) {
            rc = cnt[i].reserve(sizeof(int32_t) * tiles);
            if (rc == PB_OK) rc = off[i].reserve(sizeof(int64_t) * (tiles + 1));
        }
        if (rc != PB_OK) break;
        k_runs<false><<<(unsigned) tiles, ED_THREADS, 0, st>>>(mark.as<uint8_t>(), L, cnt[0].as<int32_t>(), cnt[1].as<int32_t>(), nullptr, nullptr,
                                                              nullptr, nullptr);
        for (int i = 0; i < 2; i++) k_scan_excl<<<1, 1024, 0, st>>>(cnt[i].as<int32_t>(), off[i].as<int64_t>(), tiles, nullptr);
        int64_t n_runs = 0;
        PB_CUDA(cudaMemcpyAsync(&n_runs, off[0].as<int64_t>() + tiles, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        *n_lines = n_runs;
        if (n_runs == 0) break;
        if ((rc = ra.reserve(sizeof(int64_t) * n_runs)) != PB_OK) break;
        if ((rc = rb.reserve(sizeof(int64_t) * n_runs)) != PB_OK) break;
        if ((rc = alt.reserve(sizeof(int64_t) * n_runs)) != PB_OK) break;
        if ((rc = tlen.reserve(sizeof(int32_t) * n_runs)) != PB_OK) break;
        if ((rc = toff.reserve(sizeof(int64_t) * (n_runs + 1))) != PB_OK) break;
        if ((rc = upload(name, contig, (size_t) name_len + 1, st)) != PB_OK) break;
        k_runs<true><<<(unsigned) tiles, ED_THREADS, 0, st>>>(mark.as<uint8_t>(), L, nullptr, nullptr, off[0].as<int64_t>(), off[1].as<int64_t>(),
                                                             ra.as<int64_t>(), rb.as<int64_t>());
        EditView V{d_events, n_events, mark.as<uint8_t>(), d_draft, span_start, L};
        const unsigned g = (unsigned) ((n_runs + 127) / 128);
        k_run_info<<<g, 128, 0, st>>>(V, ra.as<int64_t>(), rb.as<int64_t>(), n_runs, alt.as<int64_t>());
        k_run_format<false><<<g, 128, 0, st>>>(V, ra.as<int64_t>(), rb.as<int64_t>(), alt.as<int64_t>(), n_runs, name.as<char>(), name_len,
                                               tlen.as<int32_t>(), nullptr, nullptr, nullptr);
        k_scan_excl<<<1, 1024, 0, st>>>(tlen.as<int32_t>(), toff.as<int64_t>(), n_runs, nullptr);
        PB_CUDA(cudaMemcpyAsync(n_text, toff.as<int64_t>() + n_runs, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaStreamSynchronize(st));
        if (n_runs > capacity_lines || *n_text > capacity_text) {
            set_error("edits VCF capacity (%lld lines, %lld bytes) < (%lld, %lld) needed", (long long) capacity_lines,
                      (long long) capacity_text, (long long) n_runs, (long long) *n_text);
            rc = PB_ERR_CAPACITY; break;
        }
        k_run_format<true><<<g, 128, 0, st>>>(V, ra.as<int64_t>(), rb.as<int64_t>(), alt.as<int64_t>(), n_runs, name.as<char>(), name_len,
                                              nullptr, toff.as<int64_t>(), d_text, d_lines);
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("edits VCF: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    } while (0);
    DevBuf *bufs[] = {&mark, &cover, &cnt[0], &cnt[1], &off[0], &off[1], &ra, &rb, &alt, &tlen, &toff, &name};
    for (auto *x : bufs) x->release();
    return rc;
}
