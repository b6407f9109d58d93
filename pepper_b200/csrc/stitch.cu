// Polish stitch on the GPU (SURVEY 8f row f3): the reference builds a Python dict keyed by (position, index) per
// base (pepper/modules/python/Stitch.py:64-74) and sorts it; here every image column decides locally whether it survives
// (padding, region buffer, chunk-overlap winner, label 0), a scan gives its output offset, and the consensus string is
// written once.
#include "handles.cuh"
#include <algorithm>

namespace pb {

constexpr int SCOLS = 1000;
constexpr int S_OVERLAP = 50;       // SEQ_OVERLAP, pepper Options.py
constexpr int S_BUFFER = 200;       // 2 * MIN_IMAGE_OVERLAP, Stitch.py:42

// str(a) < str(b) for non-negative decimal integers (chunk ids are sorted as strings, Stitch.py:50)
__device__ bool str_less(int a, int b) {
    char sa[12], sb[12];
    int la = 0, lb = 0;
    do { sa[la++] = (char) ('0' + a % 10); a /= 10; } while (a);
    do { sb[lb++] = (char) ('0' + b % 10); b /= 10; } while (b);
    for (int i = 0; i < la && i < lb; i++) {
        const char ca = sa[la - 1 - i], cb = sb[lb - 1 - i];
        if (ca != cb) return ca < cb;
    }
    return la < lb;
}

// FASTQ quality byte of a network phred (0..100): '!' + phred clamped to 93, so that every byte is a printable FASTQ quality
__device__ __forceinline__ char qv_byte(uint8_t phred) { return (char) ('!' + (phred < 93 ? phred : 93)); }

// The columns of one image that survive (padding, region buffer, the losing side of each chunk overlap, label 0), written in
// order when WRITE: survivor o's base to out[o * stride] and, given `phred`, its QV byte to qual[o * stride] (o counted from
// o0; o < capacity).  Returns how many survive.  `st` = the start of the image's region.
template <bool WRITE>
__device__ int stitch_columns(const uint8_t *__restrict__ bases, const uint8_t *__restrict__ phred, const int64_t *__restrict__ position,
                              const int32_t *__restrict__ index, int64_t st, bool tail_lost, bool head_lost, char *out, char *qual,
                              int stride, int64_t o0, int64_t capacity) {
    __shared__ int s_warp[8];
    __shared__ int s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    int total = 0;
    for (int c0 = 0; c0 < SCOLS; c0 += 256) {
        const int c = c0 + tid;
        bool keep = false;
        uint8_t b = 0;
        if (c < SCOLS) {
            const int64_t pos = position[c];
            const int idx = index[c];
            b = bases[c];
            keep = pos >= 0 && idx >= 0 && !(st > 0 && pos <= st + S_BUFFER) && b != 0 && b <= 4;
            if (tail_lost && c >= SCOLS - S_OVERLAP) keep = false;
            if (head_lost && c < S_OVERLAP) keep = false;
        }
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        const int wcount = __popc(m), wprefix = __popc(m & ((1u << lane) - 1u));
        if (lane == 0) s_warp[warp] = wcount;
        __syncthreads();
        int base = s_carry;
        for (int w = 0; w < warp; w++) base += s_warp[w];
        if (WRITE && keep) {
            const int64_t o = o0 + base + wprefix;
            if (o < capacity) {
                out[o * stride] = "ACGT"[b - 1];
                if (phred) qual[o * stride] = qv_byte(phred[c]);
            }
        }
        __syncthreads();
        if (tid == 0) { int s = 0; for (int w = 0; w < 8; w++) s += s_warp[w]; s_carry += s; }
        __syncthreads();
        total = s_carry;
    }
    return total;
}

template <bool WRITE>
__global__ void __launch_bounds__(256) k_stitch(const uint8_t *__restrict__ bases, const uint8_t *__restrict__ phred,
                                                const int64_t *__restrict__ position, const int32_t *__restrict__ index,
                                                const int32_t *__restrict__ image_region, const int32_t *__restrict__ chunk_id,
                                                const int64_t *__restrict__ region_starts, int64_t n_images, int32_t *__restrict__ counts,
                                                const int64_t *__restrict__ offsets, char *out, char *qual, int64_t capacity) {
    const int64_t im = blockIdx.x;
    const int reg = image_region[im], cid = chunk_id[im];
    const int64_t st = region_starts[reg];
    // which side of each 50-column overlap loses (the chunk whose id sorts earlier as a string is overwritten)
    const bool has_next = (im + 1 < n_images) && image_region[im + 1] == reg;
    const bool has_prev = (im > 0) && image_region[im - 1] == reg;
    const bool tail_lost = has_next && str_less(cid, chunk_id[im + 1]);
    const bool head_lost = has_prev && !str_less(chunk_id[im - 1], cid);
    const int total = stitch_columns<WRITE>(bases + im * SCOLS, phred ? phred + im * SCOLS : nullptr, position + im * SCOLS,
                                            index + im * SCOLS, st, tail_lost, head_lost, out, qual, 1, WRITE ? offsets[im] : 0,
                                            capacity);
    if (!WRITE && threadIdx.x == 0) counts[im] = total;
}

// The edit events of one image of an edits session (pb_edit_event_t), written in order from event o0 when WRITE (o < ev_capacity).
// A column wins its (position, index) by the rule of stitch_columns with label-0 columns kept; a winner is an event when it
// is a deletion (label 0 at index 0), a substitution (label != draft base at index 0) or an insertion (index >= 1, label !=
// 0).  After the columns, one PB_EDIT_COVERAGE record: the first and last index-0 position the image won (none: no record).
// Returns the records.
template <bool WRITE>
__device__ int edit_columns(const SinkArgs &A, int64_t im, bool tail_lost, bool head_lost, int64_t o0) {
    __shared__ int s_warp[8];
    __shared__ int s_carry;
    __shared__ unsigned long long s_first, s_last;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint8_t *bases = A.bases + im * SCOLS, *phred = A.edit_phred + im * SCOLS, *draft = A.draft + im * SCOLS;
    const int64_t *position = A.position + im * SCOLS;
    const int32_t *index = A.index + im * SCOLS;
    const int64_t st = A.start[im];
    if (tid == 0) { s_carry = 0; s_first = ~0ull; s_last = 0ull; }
    __syncthreads();
    bool won0 = false;
    for (int c0 = 0; c0 < SCOLS; c0 += 256) {
        const int c = c0 + tid;
        bool ev = false;
        uint8_t b = 0;
        int64_t pos = -1;
        int idx = -1;
        if (c < SCOLS) {
            pos = position[c];
            idx = index[c];
            b = bases[c];
            bool win = pos >= 0 && idx >= 0 && !(st > 0 && pos <= st + S_BUFFER) && b <= 4;
            if (tail_lost && c >= SCOLS - S_OVERLAP) win = false;
            if (head_lost && c < S_OVERLAP) win = false;
            if (win && idx == 0) {
                won0 = true;
                atomicMin(&s_first, (unsigned long long) pos);
                atomicMax(&s_last, (unsigned long long) pos);
            }
            ev = win && (idx == 0 ? (b == 0 || (uint8_t) "ACGT"[b - 1] != draft[c]) : b != 0);
        }
        const unsigned m = __ballot_sync(0xffffffffu, ev);
        const int wcount = __popc(m), wprefix = __popc(m & ((1u << lane) - 1u));
        if (lane == 0) s_warp[warp] = wcount;
        __syncthreads();
        int base = s_carry;
        for (int w = 0; w < warp; w++) base += s_warp[w];
        if (WRITE && ev) {
            const int64_t o = o0 + base + wprefix;
            if (o < A.ev_capacity) {
                pb_edit_event_t e;
                e.position = pos; e.index = idx; e.label = b; e.phred = phred[c]; e.draft = draft[c]; e.kind = PB_EDIT_COLUMN;
                A.events[o] = e;
            }
        }
        __syncthreads();
        if (tid == 0) { int s = 0; for (int w = 0; w < 8; w++) s += s_warp[w]; s_carry += s; }
        __syncthreads();
    }
    const bool covered = __syncthreads_or(won0);
    const int total = s_carry;
    if (WRITE && covered && tid == 0 && o0 + total < A.ev_capacity) {
        pb_edit_event_t e;
        e.position = (int64_t) s_first; e.index = (int32_t) (s_last - s_first); e.label = 0; e.phred = 0; e.draft = 0;
        e.kind = PB_EDIT_COVERAGE;
        A.events[o0 + total] = e;
    }
    return total + (covered ? 1 : 0);
}

// Stitch-to-sink: the same rule over one network chunk of a streaming polish session, appended to a sink at a running record
// offset that stays on the device.  A record is one consensus byte, or with A.phred the 2 bytes (base, QV byte).  The
// neighbours that decide the overlaps may lie outside the chunk: the next image's region / chunk id come from the session's
// image metadata (known before the network runs, A.n_known images from the chunk's first one), the previous image's from
// A.prev_region / A.prev_cid.
template <bool WRITE>
__global__ void __launch_bounds__(256) k_stitch_sink(SinkArgs A) {
    const int64_t im = blockIdx.x;
    const int reg = A.region[im], cid = A.cid[im];
    const bool has_next = (im + 1 < A.n_known) && A.region[im + 1] == reg;
    const int preg = im > 0 ? A.region[im - 1] : A.prev_region, pcid = im > 0 ? A.cid[im - 1] : A.prev_cid;
    const bool tail_lost = has_next && str_less(cid, A.cid[im + 1]);
    const bool head_lost = preg == reg && !str_less(pcid, cid);
    const int total = stitch_columns<WRITE>(A.bases + im * SCOLS, A.phred ? A.phred + im * SCOLS : nullptr, A.position + im * SCOLS,
                                            A.index + im * SCOLS, A.start[im], tail_lost, head_lost, A.out,
                                            A.phred ? A.out + 1 : nullptr, A.phred ? 2 : 1, WRITE ? A.state[0] + A.offsets[im] : 0,
                                            A.capacity);
    if (!WRITE && threadIdx.x == 0) {
        A.counts[im] = total;
        if (total) atomicAdd(reinterpret_cast<unsigned long long *>(A.group_bytes + A.slot[im]), (unsigned long long) total);
    }
    if (A.events) {
        const int ne = edit_columns<WRITE>(A, im, tail_lost, head_lost, WRITE ? A.state[1] + A.ev_offsets[im] : 0);
        if (!WRITE && threadIdx.x == 0) {
            A.ev_counts[im] = ne;
            if (ne) atomicAdd(reinterpret_cast<unsigned long long *>(A.group_events + A.slot[im]), (unsigned long long) ne);
        }
    }
}

__global__ void k_sink_advance(int64_t *state, const int64_t *chunk_total) { state[0] += *chunk_total; }

// count, scan, write, advance: four launches on `st`, no host synchronisation
int polish_sink(SinkArgs A, DevBuf &counts, DevBuf &offsets, cudaStream_t st, DevBuf *ev) {
    if (A.n <= 0) return PB_OK;
    PB_TRY(counts.reserve(sizeof(int32_t) * A.n));
    PB_TRY(offsets.reserve(sizeof(int64_t) * (A.n + 1)));
    A.counts = counts.as<int32_t>();
    A.offsets = offsets.as<int64_t>();
    if (A.events) {
        if (!ev) { set_error("edits sink without scratch"); return PB_ERR_ARG; }
        PB_TRY(ev[0].reserve(sizeof(int32_t) * A.n));
        PB_TRY(ev[1].reserve(sizeof(int64_t) * (A.n + 1)));
        A.ev_counts = ev[0].as<int32_t>();
        A.ev_offsets = ev[1].as<int64_t>();
    }
    k_stitch_sink<false><<<(unsigned) A.n, 256, 0, st>>>(A);
    k_scan_excl<<<1, 1024, 0, st>>>(A.counts, offsets.as<int64_t>(), A.n, nullptr);
    if (A.events) k_scan_excl<<<1, 1024, 0, st>>>(A.ev_counts, ev[1].as<int64_t>(), A.n, nullptr);
    k_stitch_sink<true><<<(unsigned) A.n, 256, 0, st>>>(A);
    k_sink_advance<<<1, 1, 0, st>>>(A.state, offsets.as<int64_t>() + A.n);
    if (A.events) k_sink_advance<<<1, 1, 0, st>>>(A.state + 1, ev[1].as<int64_t>() + A.n);
    PB_CUDA(cudaGetLastError());
    return PB_OK;
}

}  // namespace pb

using namespace pb;

// one-shot stitch of a contig's images: bases to d_out and, given d_phred, QV bytes to d_qual (both [capacity])
static int stitch_device(const uint8_t *d_bases, const uint8_t *d_phred, const int64_t *d_position, const int32_t *d_index,
                         const int32_t *d_image_region, const int32_t *d_chunk_id, const int64_t *d_region_starts, int64_t n_images,
                         char *d_out, char *d_qual, int64_t capacity, int64_t *n_out, cudaStream_t st) {
    if (!n_out || (d_phred && !d_qual)) { set_error("null argument"); return PB_ERR_ARG; }
    *n_out = 0;
    if (n_images <= 0) return PB_OK;
    DevBuf counts, offsets;
    PB_TRY(counts.reserve(sizeof(int32_t) * n_images));
    PB_TRY(offsets.reserve(sizeof(int64_t) * (n_images + 2)));
    k_stitch<false><<<(unsigned) n_images, 256, 0, st>>>(d_bases, nullptr, d_position, d_index, d_image_region, d_chunk_id, d_region_starts,
                                                        n_images, counts.as<int32_t>(), nullptr, nullptr, nullptr, 0);
    k_scan_excl<<<1, 1024, 0, st>>>(counts.as<int32_t>(), offsets.as<int64_t>(), n_images, offsets.as<int64_t>() + n_images + 1);
    int64_t total = 0;
    PB_CUDA(cudaMemcpyAsync(&total, offsets.as<int64_t>() + n_images, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    *n_out = total;
    int rc = PB_OK;
    if (total > capacity) {
        set_error("consensus capacity %lld < %lld needed", (long long) capacity, (long long) total);
        rc = PB_ERR_CAPACITY;
    } else if (total > 0) {
        k_stitch<true><<<(unsigned) n_images, 256, 0, st>>>(d_bases, d_phred, d_position, d_index, d_image_region, d_chunk_id, d_region_starts,
                                                           n_images, nullptr, offsets.as<int64_t>(), d_out, d_qual, capacity);
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("stitch: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    }
    counts.release(); offsets.release();
    return rc;
}

static int stitch_host(const uint8_t *h_bases, const uint8_t *h_phred, const int64_t *h_position, const int32_t *h_index,
                       const int32_t *h_image_region, const int32_t *h_chunk_id, const int64_t *h_region_starts, int64_t n_regions,
                       int64_t n_images, char *h_out, char *h_qual, int64_t capacity, int64_t *n_out, cudaStream_t st) {
    if (!n_out || (h_phred && !h_qual)) { set_error("null argument"); return PB_ERR_ARG; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) { set_error("no CUDA device: libpepper_b200 has no CPU fallback"); return PB_ERR_CUDA; }
    *n_out = 0;
    if (n_images <= 0) return PB_OK;
    const size_t cap = (size_t) std::max<int64_t>(capacity, 1);
    DevBuf b, p, i, r, c, s, o, ph, q;
    PB_TRY(upload(b, h_bases, (size_t) n_images * SCOLS, st));
    PB_TRY(upload(p, h_position, sizeof(int64_t) * n_images * SCOLS, st));
    PB_TRY(upload(i, h_index, sizeof(int32_t) * n_images * SCOLS, st));
    PB_TRY(upload(r, h_image_region, sizeof(int32_t) * n_images, st));
    PB_TRY(upload(c, h_chunk_id, sizeof(int32_t) * n_images, st));
    PB_TRY(upload(s, h_region_starts, sizeof(int64_t) * n_regions, st));
    PB_TRY(o.reserve(cap));
    if (h_phred) {
        PB_TRY(upload(ph, h_phred, (size_t) n_images * SCOLS, st));
        PB_TRY(q.reserve(cap));
    }
    int rc = stitch_device(b.as<uint8_t>(), h_phred ? ph.as<uint8_t>() : nullptr, p.as<int64_t>(), i.as<int32_t>(), r.as<int32_t>(),
                           c.as<int32_t>(), s.as<int64_t>(), n_images, o.as<char>(), h_phred ? q.as<char>() : nullptr, capacity, n_out, st);
    if (rc == PB_OK && *n_out > 0) {
        cudaError_t e = cudaMemcpyAsync(h_out, o.p, (size_t) *n_out, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess && h_phred) e = cudaMemcpyAsync(h_qual, q.p, (size_t) *n_out, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("stitch copy back: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    }
    DevBuf *bufs[] = {&b, &p, &i, &r, &c, &s, &o, &ph, &q};
    for (auto *x : bufs) x->release();
    return rc;
}

extern "C" int pb_polish_stitch_device(const uint8_t *d_bases, const int64_t *d_position, const int32_t *d_index,
                                       const int32_t *d_image_region, const int32_t *d_chunk_id, const int64_t *d_region_starts,
                                       int64_t n_images, char *d_out, int64_t capacity, int64_t *n_out, void *stream_) {
    return stitch_device(d_bases, nullptr, d_position, d_index, d_image_region, d_chunk_id, d_region_starts, n_images, d_out, nullptr,
                         capacity, n_out, (cudaStream_t) stream_);
}

extern "C" int pb_polish_stitch_qual_device(const uint8_t *d_bases, const uint8_t *d_phred, const int64_t *d_position,
                                            const int32_t *d_index, const int32_t *d_image_region, const int32_t *d_chunk_id,
                                            const int64_t *d_region_starts, int64_t n_images, char *d_out, char *d_qual,
                                            int64_t capacity, int64_t *n_out, void *stream_) {
    if (!d_phred) { set_error("null argument"); return PB_ERR_ARG; }
    return stitch_device(d_bases, d_phred, d_position, d_index, d_image_region, d_chunk_id, d_region_starts, n_images, d_out, d_qual,
                         capacity, n_out, (cudaStream_t) stream_);
}

extern "C" int pb_polish_stitch_host(const uint8_t *h_bases, const int64_t *h_position, const int32_t *h_index,
                                     const int32_t *h_image_region, const int32_t *h_chunk_id, const int64_t *h_region_starts,
                                     int64_t n_regions, int64_t n_images, char *h_out, int64_t capacity, int64_t *n_out, void *stream_) {
    return stitch_host(h_bases, nullptr, h_position, h_index, h_image_region, h_chunk_id, h_region_starts, n_regions, n_images, h_out,
                       nullptr, capacity, n_out, (cudaStream_t) stream_);
}

extern "C" int pb_polish_stitch_qual_host(const uint8_t *h_bases, const uint8_t *h_phred, const int64_t *h_position,
                                          const int32_t *h_index, const int32_t *h_image_region, const int32_t *h_chunk_id,
                                          const int64_t *h_region_starts, int64_t n_regions, int64_t n_images, char *h_out,
                                          char *h_qual, int64_t capacity, int64_t *n_out, void *stream_) {
    if (!h_phred) { set_error("null argument"); return PB_ERR_ARG; }
    return stitch_host(h_bases, h_phred, h_position, h_index, h_image_region, h_chunk_id, h_region_starts, n_regions, n_images, h_out,
                       h_qual, capacity, n_out, (cudaStream_t) stream_);
}

// diagnostics: host predictions (images in session order) through the stitch-to-sink kernel `chunk` images at a time, the way a
// streaming session feeds it one network chunk after the other.  h_region_bytes (optional): records per region [n_regions].
// Given h_phred, h_out holds 2-byte (base, QV byte) records [capacity].  Given h_draft (and h_ev_phred), the event sink of an
// edits session: h_events [ev_capacity], *n_events, h_region_events (optional) [n_regions].
struct EditTest {
    const uint8_t *h_phred = nullptr, *h_draft = nullptr;
    pb_edit_event_t *h_events = nullptr; int64_t capacity = 0; int64_t *n_events = nullptr, *h_region_events = nullptr;
};
static int stitch_sink_test(const uint8_t *h_bases, const uint8_t *h_phred, const int64_t *h_position, const int32_t *h_index,
                            const int32_t *h_image_region, const int32_t *h_chunk_id, const int64_t *h_region_starts,
                            int64_t n_regions, int64_t n_images, int64_t chunk, char *h_out, int64_t capacity,
                            int64_t *n_out, int64_t *h_region_bytes, cudaStream_t st, const EditTest &E = EditTest()) {
    const bool edits = E.h_draft != nullptr;
    if (!n_out || chunk <= 0 || n_regions <= 0) { set_error("bad argument"); return PB_ERR_ARG; }
    if (edits && (!E.h_phred || !E.n_events || (E.capacity > 0 && !E.h_events))) { set_error("null argument"); return PB_ERR_ARG; }
    if (edits) *E.n_events = 0;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) { set_error("no CUDA device: libpepper_b200 has no CPU fallback"); return PB_ERR_CUDA; }
    *n_out = 0;
    if (n_images <= 0) return PB_OK;
    const size_t rec = h_phred ? 2 : 1;
    std::vector<int64_t> start((size_t) n_images);
    for (int64_t i = 0; i < n_images; i++) {
        if (h_image_region[i] < 0 || h_image_region[i] >= n_regions) { set_error("image %lld: region out of range", (long long) i); return PB_ERR_ARG; }
        start[i] = h_region_starts[h_image_region[i]];
    }
    DevBuf b, ph, p, i, r, c, s, o, state, gb, counts, offsets, eph, dr, evo, ge, evs[2];
    int rc = PB_OK;
    do {
        if ((rc = upload(b, h_bases, (size_t) n_images * SCOLS, st)) != PB_OK) break;
        if (h_phred && (rc = upload(ph, h_phred, (size_t) n_images * SCOLS, st)) != PB_OK) break;
        if ((rc = upload(p, h_position, sizeof(int64_t) * n_images * SCOLS, st)) != PB_OK) break;
        if ((rc = upload(i, h_index, sizeof(int32_t) * n_images * SCOLS, st)) != PB_OK) break;
        if ((rc = upload(r, h_image_region, sizeof(int32_t) * n_images, st)) != PB_OK) break;
        if ((rc = upload(c, h_chunk_id, sizeof(int32_t) * n_images, st)) != PB_OK) break;
        if ((rc = upload(s, start.data(), sizeof(int64_t) * n_images, st)) != PB_OK) break;
        if ((rc = o.reserve(rec * (size_t) std::max<int64_t>(capacity, 1))) != PB_OK) break;
        if ((rc = state.reserve(2 * sizeof(int64_t))) != PB_OK) break;
        if ((rc = gb.reserve(sizeof(int64_t) * n_regions)) != PB_OK) break;
        if (edits) {
            if ((rc = upload(eph, E.h_phred, (size_t) n_images * SCOLS, st)) != PB_OK) break;
            if ((rc = upload(dr, E.h_draft, (size_t) n_images * SCOLS, st)) != PB_OK) break;
            if ((rc = evo.reserve(sizeof(pb_edit_event_t) * (size_t) std::max<int64_t>(E.capacity, 1))) != PB_OK) break;
            if ((rc = ge.reserve(sizeof(int64_t) * n_regions)) != PB_OK) break;
            if (cudaMemsetAsync(ge.p, 0, sizeof(int64_t) * n_regions, st) != cudaSuccess) { set_error("memset failed"); rc = PB_ERR_CUDA; break; }
        }
        if (cudaMemsetAsync(state.p, 0, 2 * sizeof(int64_t), st) != cudaSuccess || cudaMemsetAsync(gb.p, 0, sizeof(int64_t) * n_regions, st) != cudaSuccess) {
            set_error("memset failed"); rc = PB_ERR_CUDA; break;
        }
        for (int64_t c0 = 0; c0 < n_images && rc == PB_OK; c0 += chunk) {
            SinkArgs A;
            A.n = std::min(chunk, n_images - c0); A.n_known = n_images - c0;
            A.bases = b.as<uint8_t>() + c0 * SCOLS; A.position = p.as<int64_t>() + c0 * SCOLS; A.index = i.as<int32_t>() + c0 * SCOLS;
            A.phred = h_phred ? ph.as<uint8_t>() + c0 * SCOLS : nullptr;
            A.region = r.as<int32_t>() + c0; A.cid = c.as<int32_t>() + c0; A.start = s.as<int64_t>() + c0; A.slot = r.as<int32_t>() + c0;
            A.prev_region = c0 > 0 ? h_image_region[c0 - 1] : -1; A.prev_cid = c0 > 0 ? h_chunk_id[c0 - 1] : 0;
            A.state = state.as<int64_t>(); A.group_bytes = gb.as<int64_t>(); A.out = o.as<char>(); A.capacity = capacity;
            if (edits) {
                A.edit_phred = eph.as<uint8_t>() + c0 * SCOLS; A.draft = dr.as<uint8_t>() + c0 * SCOLS;
                A.events = evo.as<pb_edit_event_t>(); A.ev_capacity = E.capacity; A.group_events = ge.as<int64_t>();
            }
            rc = polish_sink(A, counts, offsets, st, evs);
        }
        if (rc != PB_OK) break;
        int64_t total = 0;
        cudaError_t e = cudaMemcpyAsync(&total, state.p, sizeof(int64_t), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess && h_region_bytes) e = cudaMemcpyAsync(h_region_bytes, gb.p, sizeof(int64_t) * n_regions, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("stitch sink: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; break; }
        *n_out = total;
        int64_t n_ev = 0;
        if (edits) {
            e = cudaMemcpyAsync(&n_ev, state.as<int64_t>() + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess && E.h_region_events) e = cudaMemcpyAsync(E.h_region_events, ge.p, sizeof(int64_t) * n_regions, cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            if (e != cudaSuccess) { set_error("stitch sink: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; break; }
            *E.n_events = n_ev;
        }
        if (total > capacity) { set_error("consensus capacity %lld < %lld needed", (long long) capacity, (long long) total); rc = PB_ERR_CAPACITY; break; }
        if (n_ev > E.capacity) { set_error("edit event capacity %lld < %lld needed", (long long) E.capacity, (long long) n_ev); rc = PB_ERR_CAPACITY; break; }
        if (total > 0) e = cudaMemcpyAsync(h_out, o.p, rec * (size_t) total, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess && n_ev > 0) e = cudaMemcpyAsync(E.h_events, evo.p, sizeof(pb_edit_event_t) * (size_t) n_ev, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("stitch sink copy back: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    } while (0);
    DevBuf *bufs[] = {&b, &ph, &p, &i, &r, &c, &s, &o, &state, &gb, &counts, &offsets, &eph, &dr, &evo, &ge, &evs[0], &evs[1]};
    for (auto *x : bufs) x->release();
    return rc;
}

extern "C" int pb_test_polish_stitch_sink(const uint8_t *h_bases, const int64_t *h_position, const int32_t *h_index,
                                          const int32_t *h_image_region, const int32_t *h_chunk_id, const int64_t *h_region_starts,
                                          int64_t n_regions, int64_t n_images, int64_t chunk, char *h_out, int64_t capacity,
                                          int64_t *n_out, int64_t *h_region_bytes, void *stream_) {
    return stitch_sink_test(h_bases, nullptr, h_position, h_index, h_image_region, h_chunk_id, h_region_starts, n_regions, n_images, chunk,
                            h_out, capacity, n_out, h_region_bytes, (cudaStream_t) stream_);
}

extern "C" int pb_test_polish_stitch_sink_qual(const uint8_t *h_bases, const uint8_t *h_phred, const int64_t *h_position,
                                               const int32_t *h_index, const int32_t *h_image_region, const int32_t *h_chunk_id,
                                               const int64_t *h_region_starts, int64_t n_regions, int64_t n_images, int64_t chunk,
                                               char *h_records, int64_t capacity, int64_t *n_out, int64_t *h_region_records,
                                               void *stream_) {
    if (!h_phred) { set_error("null argument"); return PB_ERR_ARG; }
    return stitch_sink_test(h_bases, h_phred, h_position, h_index, h_image_region, h_chunk_id, h_region_starts, n_regions, n_images, chunk,
                            h_records, capacity, n_out, h_region_records, (cudaStream_t) stream_);
}

extern "C" int pb_test_polish_stitch_sink_edits(const uint8_t *h_bases, const uint8_t *h_phred, const uint8_t *h_draft,
                                                const int64_t *h_position, const int32_t *h_index, const int32_t *h_image_region,
                                                const int32_t *h_chunk_id, const int64_t *h_region_starts, int64_t n_regions,
                                                int64_t n_images, int64_t chunk, char *h_records, int64_t capacity, int64_t *n_out,
                                                int64_t *h_region_records, pb_edit_event_t *h_events, int64_t capacity_events,
                                                int64_t *n_events, int64_t *h_region_events, void *stream_) {
    if (!h_draft || !h_phred) { set_error("null argument"); return PB_ERR_ARG; }
    EditTest E;
    E.h_phred = h_phred; E.h_draft = h_draft; E.h_events = h_events; E.capacity = capacity_events; E.n_events = n_events;
    E.h_region_events = h_region_events;
    return stitch_sink_test(h_bases, nullptr, h_position, h_index, h_image_region, h_chunk_id, h_region_starts, n_regions, n_images, chunk,
                            h_records, capacity, n_out, h_region_records, (cudaStream_t) stream_, E);
}
