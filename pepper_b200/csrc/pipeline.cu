// Fused make_images + inference entry points (the path `pepper_variant call_variant` steps 1+2 and
// `pepper polish` steps 1+2 take, without the intermediate image HDF5 files): encoder output stays in HBM and
// feeds the network directly.
#include "handles.cuh"
#include <algorithm>
#include <vector>
#include <stdint.h>

using namespace pb;

namespace pb {

// AlignmentSummarizer.chunk_images (pepper AlignmentSummarizer.py:19-56) on the device:
// image k = columns [start, start+nvalid) of its region, zero padded to 1000, positions padded with (-1,-1)
struct ChunkRow { int64_t col_start; int32_t nvalid; int32_t region; int32_t chunk_id; int32_t pad; };

__global__ void k_polish_chunk(const ChunkRow *__restrict__ rows, const uint8_t *__restrict__ image, const int64_t *__restrict__ pos,
                               const int32_t *__restrict__ idx, uint8_t *__restrict__ imgs, int64_t *__restrict__ position,
                               int32_t *__restrict__ index, int32_t *__restrict__ iregion, int32_t *__restrict__ cid,
                               uint8_t *__restrict__ draft = nullptr, const char *__restrict__ ref = nullptr,
                               const pb_region_t *__restrict__ regions = nullptr, int32_t region0 = 0) {
    const int64_t k = blockIdx.x;
    const ChunkRow r = rows[k];
    for (int i = threadIdx.x; i < PB_POLISH_SEQ_LEN * PB_POLISH_FEATURES; i += blockDim.x) {
        const int c = i / PB_POLISH_FEATURES;
        imgs[k * PB_POLISH_SEQ_LEN * PB_POLISH_FEATURES + i] = (c < r.nvalid) ? image[(r.col_start + c) * PB_POLISH_FEATURES + (i - c * PB_POLISH_FEATURES)] : 0;
    }
    for (int c = threadIdx.x; c < PB_POLISH_SEQ_LEN; c += blockDim.x) {
        position[k * PB_POLISH_SEQ_LEN + c] = (c < r.nvalid) ? pos[r.col_start + c] : -1;
        index[k * PB_POLISH_SEQ_LEN + c] = (c < r.nvalid) ? idx[r.col_start + c] : -1;
    }
    // an edits session: each column's upper-cased draft base, from the region's reference string
    if (draft) {
        const pb_region_t rg = regions[r.region - region0];
        for (int c = threadIdx.x; c < PB_POLISH_SEQ_LEN; c += blockDim.x) {
            const int64_t o = (c < r.nvalid) ? pos[r.col_start + c] - rg.ref_start : -1;
            char b = (o >= 0 && o < rg.ref_len) ? ref[rg.ref_off + o] : 0;
            if (b >= 'a' && b <= 'z') b = (char) (b - 32);
            draft[k * PB_POLISH_SEQ_LEN + c] = (uint8_t) b;
        }
    }
    if (threadIdx.x == 0) { iregion[k] = r.region; cid[k] = r.chunk_id; }
}

}  // namespace pb

static int ensure_events(cudaEvent_t *ev, int n) {
    for (int i = 0; i < n; i++) if (!ev[i]) PB_CUDA(cudaEventCreate(&ev[i]));
    return PB_OK;
}

extern "C" int pb_variant_call_device(pb_variant_encoder_t *enc, pb_variant_net_t *net, const pb_reads_t *d_reads,
                                      const pb_region_t *d_regions, int64_t n_regions, const pb_region_t *h_regions,
                                      const char *d_ref, int64_t ref_bytes, const pb_variant_params_t *params,
                                      int64_t capacity, int8_t *d_images, int64_t *d_positions, uint8_t *d_depths,
                                      uint8_t *d_freqs, char *d_keys, int32_t *d_region_of, float *d_probs,
                                      int64_t *n_out, void *stream_) {
    if (!enc || !net) { set_error("null handle"); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    PB_TRY(ensure_events(enc->pevt, 3));
    PB_CUDA(cudaEventRecord(enc->pevt[0], st));
    PB_TRY(pb_variant_encode_device(enc, d_reads, d_regions, n_regions, h_regions, d_ref, ref_bytes, params, capacity,
                                    d_images, d_positions, d_depths, d_freqs, d_keys, d_region_of, nullptr, n_out, stream_));
    PB_CUDA(cudaEventRecord(enc->pevt[1], st));
    PB_TRY(pb_variant_net_forward_device(net, d_images, *n_out, d_probs, nullptr, stream_));
    PB_CUDA(cudaEventRecord(enc->pevt[2], st));
    PB_CUDA(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&enc->pms[0], enc->pevt[0], enc->pevt[1]);
    cudaEventElapsedTime(&enc->pms[1], enc->pevt[1], enc->pevt[2]);
    return PB_OK;
}

// One group of regions [g0, g1) staged into buffer set `b` on the copy stream.  Read / reference arrays keep their
// ABSOLUTE offsets: the device base pointers are shifted back by the slice start ("virtual base"), so seq_off /
// cigar_off / ref_off need no rebasing; only the per-read arrays are re-indexed from the group's first read.
struct GroupView {
    pb_reads_t d; const pb_region_t *d_regions; const char *d_ref; std::vector<pb_region_t> h_regions;
    std::vector<int64_t> owned_end;      // gVCF track session: each region's last owned position (pb_variant_stream_owned)
};

static int stage_group(pb_variant_encoder_t *e, int b, const pb_reads_t *h, const pb_region_t *h_regions, int64_t g0, int64_t g1,
                       const char *h_ref, GroupView &V) {
    cudaStream_t cs = e->copy_stream;
    DevBuf *B = e->g_buf[b];
    const int64_t r0 = h_regions[g0].read_begin, r1 = h_regions[g1 - 1].read_end;
    const int64_t n = r1 - r0;
    const int64_t nb0 = h->seq_off[r0], nb1 = h->seq_off[r1], c0 = h->cigar_off[r0], c1 = h->cigar_off[r1];
    const int64_t sb0 = nb0 >> 1, sb1 = (nb1 + 1) >> 1;
    PB_TRY(upload(B[0], h->pos + r0, sizeof(int64_t) * n, cs));
    PB_TRY(upload(B[1], h->seq_off + r0, sizeof(int64_t) * (n + 1), cs));
    PB_TRY(upload(B[2], h->cigar_off + r0, sizeof(int64_t) * (n + 1), cs));
    PB_TRY(upload(B[3], h->flags + r0, n, cs));
    PB_TRY(upload(B[4], h->mapq + r0, n, cs));
    PB_TRY(upload(B[5], h->seq + sb0, (size_t) (sb1 - sb0), cs));
    PB_TRY(upload(B[6], h->qual + nb0, (size_t) (nb1 - nb0), cs));
    PB_TRY(upload(B[7], h->cigar + c0, sizeof(uint32_t) * (c1 - c0), cs));
    V.h_regions.assign(h_regions + g0, h_regions + g1);
    int64_t ref0 = INT64_MAX, ref1 = 0;
    for (auto &rg : V.h_regions) {
        rg.read_begin -= r0; rg.read_end -= r0;
        ref0 = std::min(ref0, rg.ref_off); ref1 = std::max(ref1, rg.ref_off + rg.ref_len);
    }
    if (ref1 < ref0) { ref0 = 0; ref1 = 0; }
    PB_TRY(upload(B[8], V.h_regions.data(), sizeof(pb_region_t) * V.h_regions.size(), cs));
    PB_TRY(upload(B[9], h_ref + ref0, (size_t) (ref1 - ref0), cs));
    PB_CUDA(cudaEventRecord(e->copied[b], cs));
    V.d.n_reads = n;
    V.d.pos = B[0].as<int64_t>(); V.d.seq_off = B[1].as<int64_t>(); V.d.cigar_off = B[2].as<int64_t>();
    V.d.flags = B[3].as<uint8_t>(); V.d.mapq = B[4].as<uint8_t>();
    V.d.seq = B[5].as<uint8_t>() - sb0; V.d.qual = B[6].as<uint8_t>() - nb0; V.d.cigar = B[7].as<uint32_t>() - c0;
    V.d_regions = B[8].as<pb_region_t>();
    V.d_ref = B[9].as<char>() - ref0;
    return PB_OK;
}

__global__ void k_add_offset_i32(int32_t *p, int64_t n, int32_t off) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] += off;
}

// single-shot host entry: everything copied up front (small batches, or regions whose read ranges are not ascending)
static int variant_call_host_single(pb_variant_encoder_t *e, pb_variant_net_t *net, const pb_reads_t *h_reads,
                                    const pb_region_t *h_regions, int64_t n_regions, const char *h_ref, int64_t ref_bytes,
                                    const pb_variant_params_t *params, int64_t capacity, int8_t *h_images,
                                    int64_t *h_positions, uint8_t *h_depths, uint8_t *h_freqs, char *h_keys,
                                    int32_t *h_region_of, float *h_probs, int64_t *n_out, void *stream_) {
    cudaStream_t st = (cudaStream_t) stream_;
    DevBuf *rb[8] = {&e->h_pos, &e->h_seq_off, &e->h_cigar_off, &e->h_flags, &e->h_mapq, &e->h_seq, &e->h_qual, &e->h_cigar};
    pb_reads_t d;
    PB_TRY(upload_reads(h_reads, rb, &d, st));
    PB_TRY(upload(e->h_regions, h_regions, sizeof(pb_region_t) * n_regions, st));
    PB_TRY(upload(e->h_ref, h_ref, (size_t) ref_bytes, st));
    const int64_t cap = std::max<int64_t>(capacity, 1);
    PB_TRY(e->p_images.reserve((size_t) cap * 33 * 26));
    PB_TRY(e->p_positions.reserve(sizeof(int64_t) * cap));
    PB_TRY(e->p_depths.reserve(cap));
    PB_TRY(e->p_freqs.reserve(cap));
    PB_TRY(e->p_keys.reserve((size_t) cap * PB_ALLELE_STRIDE));
    PB_TRY(e->p_region_of.reserve(sizeof(int32_t) * cap));
    PB_TRY(e->p_probs.reserve(sizeof(float) * 3 * cap));
    PB_TRY(pb_variant_call_device(e, net, &d, e->h_regions.as<pb_region_t>(), n_regions, h_regions, e->h_ref.as<char>(), ref_bytes,
                                  params, capacity, e->p_images.as<int8_t>(), e->p_positions.as<int64_t>(), e->p_depths.as<uint8_t>(),
                                  e->p_freqs.as<uint8_t>(), e->p_keys.as<char>(), e->p_region_of.as<int32_t>(), e->p_probs.as<float>(),
                                  n_out, stream_));
    const int64_t n = *n_out;
    if (n > 0) {
        if (h_images) PB_CUDA(cudaMemcpyAsync(h_images, e->p_images.p, (size_t) n * 33 * 26, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_positions, e->p_positions.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_depths, e->p_depths.p, n, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_freqs, e->p_freqs.p, n, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_keys, e->p_keys.p, (size_t) n * PB_ALLELE_STRIDE, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_region_of, e->p_region_of.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_probs, e->p_probs.p, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, st));
    }
    PB_CUDA(cudaStreamSynchronize(st));
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------- streaming session
// The unit of work is a GROUP of regions.  A session accumulates the candidates of the groups pushed so far in the
// library's device buffers, runs the network over WHOLE 9,472-candidate chunks of the accumulated candidates as they fill
// (the remainder rides along to the next group, so only the very last chunk of a session is partial), and lets the caller
// stage group g+1 (copy stream, pinned source) while the kernels of group g run.  pb_variant_call_host is a session over a
// fixed group list; the multi-GPU callers (pepper_b200/dist.py) push whatever group a rank claims next.
constexpr int64_t CALL_GROUP = 96;
constexpr int64_t CALL_FIRST_GROUP = 24;

// network chunk of the pipelined host entry == VARIANT_CHUNK of nets.cu (66 row tiles of 128 candidates)
static constexpr int64_t PIPE_NET_CHUNK = 8448;

namespace pb {
struct VariantStream {
    bool active = false;
    pb_variant_params_t params;
    int64_t capacity = 0, done = 0, net_done = 0;
    pb_pred_record_t *d_records = nullptr;
    cudaStream_t st = nullptr;
    GroupView V[2];
    int32_t region_id0[2] = {0, 0};
    bool staged[2] = {false, false}, from_host[2] = {false, false};
    int next_stage = 0, next_run = 0;
    // one event triple per group (encoder start, encoder end = network start, network end): read back at _sync / _end only, so
    // that run(g+1) — whose host-side table building is not short — can start while the network of group g is still running
    std::vector<cudaEvent_t> ev;
    int64_t ev_done = 0;               // groups whose times have been added to enc_ms / net_ms
    float enc_ms = 0.f, net_ms = 0.f;
    float enc_phase_ms[5] = {0, 0, 0, 0, 0};        // prefix, count, sites, alleles, windows — summed over the groups
    int64_t enc_launches = 0, net_launches = 0, groups = 0;
    // gVCF track (pb_variant_stream_track): uint32 [track_cap], filled in run order; track_reg holds the running group's
    // (track offset, owned end) per region
    uint32_t *d_track = nullptr;
    int64_t track_cap = 0, track_done = 0, track_need = 0;    // track_need > track_cap: a group did not fit
    DevBuf track_reg;
    std::vector<int64_t> h_track_reg;
};
}  // namespace pb

static int session(pb_variant_encoder_t *e, VariantStream **S, bool need_active) {
    if (!e) { set_error("null handle"); return PB_ERR_ARG; }
    if (!e->vstream) e->vstream = new VariantStream();
    *S = e->vstream;
    if (need_active && !(*S)->active) { set_error("no active stream session: call pb_variant_stream_begin first"); return PB_ERR_STATE; }
    return PB_OK;
}

extern "C" int pb_variant_stream_begin(pb_variant_encoder_t *e, pb_variant_net_t *net, const pb_variant_params_t *params,
                                       int64_t capacity, pb_pred_record_t *d_records, void *stream_) {
    if (!e || !net || !params) { set_error("null argument"); return PB_ERR_ARG; }
    VariantStream *S;
    PB_TRY(session(e, &S, false));
    PB_CUDA(cudaSetDevice(e->device));
    if (!e->copy_stream) {
        PB_CUDA(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
        for (int b = 0; b < 2; b++) PB_CUDA(cudaEventCreateWithFlags(&e->copied[b], cudaEventDisableTiming));
    }
    PB_TRY(ensure_events(e->pevt, 3));
    const int64_t cap = std::max<int64_t>(capacity, 1);
    PB_TRY(e->p_images.reserve((size_t) cap * 33 * 26));
    PB_TRY(e->p_positions.reserve(sizeof(int64_t) * cap));
    PB_TRY(e->p_depths.reserve(cap));
    PB_TRY(e->p_freqs.reserve(cap));
    PB_TRY(e->p_keys.reserve((size_t) cap * PB_ALLELE_STRIDE));
    PB_TRY(e->p_region_of.reserve(sizeof(int32_t) * cap));
    PB_TRY(e->p_probs.reserve(sizeof(float) * 3 * cap));
    S->active = true; S->params = *params; S->capacity = capacity; S->done = 0; S->net_done = 0; S->d_records = d_records;
    S->st = (cudaStream_t) stream_;
    S->staged[0] = S->staged[1] = false; S->next_stage = 0; S->next_run = 0; S->ev_done = 0;
    S->enc_ms = S->net_ms = 0.f;
    for (int i = 0; i < 5; i++) S->enc_phase_ms[i] = 0.f;
    S->enc_launches = S->net_launches = S->groups = 0;
    S->d_track = nullptr; S->track_cap = 0; S->track_done = 0; S->track_need = 0;
    for (int b = 0; b < 2; b++) S->V[b].owned_end.clear();
    return PB_OK;
}

// gVCF track of the session begun last: call before the first stage
extern "C" int pb_variant_stream_track(pb_variant_encoder_t *e, int64_t capacity_positions, uint32_t *d_track) {
    VariantStream *S;
    PB_TRY(session(e, &S, true));
    if (!d_track || capacity_positions < 0) { set_error("bad track"); return PB_ERR_ARG; }
    if (S->groups > 0 || S->staged[0] || S->staged[1]) { set_error("attach the track before the first stage"); return PB_ERR_STATE; }
    S->d_track = d_track; S->track_cap = capacity_positions; S->track_done = 0; S->track_need = 0;
    return PB_OK;
}

// owned ends of the group staged last (one per region, absolute, inclusive): its regions' track rows are [cand_start, owned_end]
extern "C" int pb_variant_stream_owned(pb_variant_encoder_t *e, const int64_t *h_owned_end, int64_t n) {
    VariantStream *S;
    PB_TRY(session(e, &S, true));
    if (!S->d_track) { set_error("no track attached"); return PB_ERR_STATE; }
    const int b = S->next_stage ^ 1;
    GroupView &V = S->V[b];
    if (!S->staged[b] || !h_owned_end || n != (int64_t) V.h_regions.size()) { set_error("owned ends do not match the staged group"); return PB_ERR_ARG; }
    for (int64_t r = 0; r < n; r++)
        if (h_owned_end[r] < V.h_regions[r].cand_start - 1 || h_owned_end[r] > V.h_regions[r].cand_end) {
            set_error("region %lld: owned end %lld outside [cand_start - 1, cand_end]", (long long) r, (long long) h_owned_end[r]);
            return PB_ERR_ARG;
        }
    V.owned_end.assign(h_owned_end, h_owned_end + n);
    return PB_OK;
}

// *n_positions = track positions written so far; *n_needed = positions the groups run or refused so far needed (above the
// capacity after a run() that returned PB_ERR_CAPACITY for the track)
extern "C" int pb_variant_stream_track_used(pb_variant_encoder_t *e, int64_t *n_positions, int64_t *n_needed) {
    VariantStream *S;
    PB_TRY(session(e, &S, false));
    if (!n_positions) { set_error("null argument"); return PB_ERR_ARG; }
    *n_positions = S->track_done;
    if (n_needed) *n_needed = std::max(S->track_done, S->track_need);
    return PB_OK;
}

// stage regions [g0, g1) of a host-resident workload into the free staging buffer (asynchronous H2D on the copy stream)
extern "C" int pb_variant_stream_stage_host(pb_variant_encoder_t *e, const pb_reads_t *h_reads, const pb_region_t *h_regions,
                                            int64_t g0, int64_t g1, const char *h_ref, int32_t region_id0) {
    VariantStream *S;
    PB_TRY(session(e, &S, true));
    if (!h_reads || !h_regions || g0 < 0 || g1 <= g0) { set_error("bad group [%lld, %lld)", (long long) g0, (long long) g1); return PB_ERR_ARG; }
    const int b = S->next_stage;
    if (S->staged[b]) { set_error("both staging buffers are in use: run a staged group first"); return PB_ERR_STATE; }
    for (int64_t r = g0; r < g1; r++) {
        if (h_regions[r].read_begin < 0 || h_regions[r].read_end > h_reads->n_reads || h_regions[r].read_begin > h_regions[r].read_end ||
            (r > g0 && h_regions[r].read_begin < h_regions[r - 1].read_end)) {
            set_error("region %lld: read range out of bounds or not ascending", (long long) r);
            return PB_ERR_ARG;
        }
    }
    PB_TRY(stage_group(e, b, h_reads, h_regions, g0, g1, h_ref, S->V[b]));
    S->staged[b] = true; S->from_host[b] = true; S->region_id0[b] = region_id0; S->next_stage = b ^ 1;
    return PB_OK;
}

// the same for a workload that is already resident in HBM: no copies of the reads, only the re-based region rows
extern "C" int pb_variant_stream_stage_device(pb_variant_encoder_t *e, const pb_reads_t *d_reads, const pb_region_t *h_regions,
                                              int64_t g0, int64_t g1, const char *d_ref, int32_t region_id0) {
    VariantStream *S;
    PB_TRY(session(e, &S, true));
    if (!d_reads || !h_regions || g0 < 0 || g1 <= g0) { set_error("bad group [%lld, %lld)", (long long) g0, (long long) g1); return PB_ERR_ARG; }
    const int b = S->next_stage;
    if (S->staged[b]) { set_error("both staging buffers are in use: run a staged group first"); return PB_ERR_STATE; }
    GroupView &V = S->V[b];
    const int64_t r0 = h_regions[g0].read_begin, r1 = h_regions[g1 - 1].read_end;
    if (r0 < 0 || r1 > d_reads->n_reads || r1 < r0) { set_error("group read range out of bounds"); return PB_ERR_ARG; }
    V.h_regions.assign(h_regions + g0, h_regions + g1);
    for (auto &rg : V.h_regions) { rg.read_begin -= r0; rg.read_end -= r0; }
    PB_TRY(upload(e->g_buf[b][8], V.h_regions.data(), sizeof(pb_region_t) * V.h_regions.size(), e->copy_stream));
    PB_CUDA(cudaEventRecord(e->copied[b], e->copy_stream));
    V.d = *d_reads;
    V.d.n_reads = r1 - r0;
    V.d.pos += r0; V.d.seq_off += r0; V.d.cigar_off += r0; V.d.flags += r0; V.d.mapq += r0;     // seq / qual / cigar keep absolute offsets
    V.d_regions = e->g_buf[b][8].as<pb_region_t>();
    V.d_ref = d_ref;
    S->staged[b] = true; S->from_host[b] = false; S->region_id0[b] = region_id0; S->next_stage = b ^ 1;
    return PB_OK;
}

// adds the times of every group whose events have completed (call after a stream synchronisation)
template <class Session>
static void stream_collect_timing(Session *S) {
    for (; S->ev_done < S->groups; S->ev_done++) {
        float a = 0.f, b = 0.f;
        cudaEvent_t *E = &S->ev[(size_t) 3 * S->ev_done];
        cudaEventElapsedTime(&a, E[0], E[1]);
        cudaEventElapsedTime(&b, E[1], E[2]);
        S->enc_ms += a; S->net_ms += b;
    }
}
template <class Session>
static int stream_events(Session *S, int64_t group, cudaEvent_t **E) {
    while ((int64_t) S->ev.size() < 3 * (group + 1)) {
        cudaEvent_t x;
        PB_CUDA(cudaEventCreate(&x));
        S->ev.push_back(x);
    }
    *E = &S->ev[(size_t) 3 * group];
    return PB_OK;
}

static int stream_network(pb_variant_encoder_t *e, pb_variant_net_t *net, VariantStream *S, int64_t run) {
    if (run <= 0) return PB_OK;
    pb_candidate_columns_t cols{e->p_positions.as<int64_t>() + S->net_done, e->p_region_of.as<int32_t>() + S->net_done,
                                e->p_depths.as<uint8_t>() + S->net_done, e->p_freqs.as<uint8_t>() + S->net_done,
                                e->p_keys.as<char>() + S->net_done * PB_ALLELE_STRIDE};
    PB_TRY(pb_variant_net_forward_records_device(net, e->p_images.as<int8_t>() + S->net_done * 33 * 26, run, e->p_probs.as<float>() + S->net_done * 3,
                                                 &cols, S->d_records ? S->d_records + S->net_done : nullptr, (void *) S->st));
    S->net_done += run;
    int64_t nl = 0;
    pb_variant_net_launches(net, &nl);
    S->net_launches += nl;
    return PB_OK;
}

// Encode the oldest staged group behind the accumulated candidates and queue the network over the whole chunks available
// (`flush` != 0: over everything, partial tail included).  Returns with the network still running: stage the next group, then
// call pb_variant_stream_sync.  On PB_ERR_CAPACITY *n_total holds the candidates needed so far (this group included).
extern "C" int pb_variant_stream_run(pb_variant_encoder_t *e, pb_variant_net_t *net, int flush, int64_t *n_total) {
    VariantStream *S;
    PB_TRY(session(e, &S, true));
    if (!net) { set_error("null handle"); return PB_ERR_ARG; }
    const int b = S->next_run;
    if (!S->staged[b]) { set_error("no staged group"); return PB_ERR_STATE; }
    cudaStream_t st = S->st;
    cudaEvent_t *E;
    PB_TRY(stream_events(S, S->groups, &E));
    PB_CUDA(cudaStreamWaitEvent(st, e->copied[b], 0));
    GroupView &V = S->V[b];
    int64_t n_g = 0;
    const int64_t done = S->done, room = std::max<int64_t>(S->capacity - done, 0);
    int64_t track_need = 0;
    if (S->d_track) {
        const int64_t nr = (int64_t) V.h_regions.size();
        if ((int64_t) V.owned_end.size() != nr) { set_error("gVCF track session: call pb_variant_stream_owned after each stage"); return PB_ERR_STATE; }
        S->h_track_reg.resize((size_t) 2 * nr);
        for (int64_t r = 0; r < nr; r++) {
            S->h_track_reg[2 * r] = S->track_done + track_need;
            S->h_track_reg[2 * r + 1] = V.owned_end[r];
            track_need += V.owned_end[r] - V.h_regions[r].cand_start + 1;
        }
        if (S->track_done + track_need > S->track_cap) {
            S->track_need = S->track_done + track_need;
            S->staged[b] = false; S->next_run = b ^ 1;
            if (n_total) *n_total = done;
            cudaStreamSynchronize(e->copy_stream);
            set_error("gVCF track capacity %lld positions < %lld needed", (long long) S->track_cap, (long long) (S->track_done + track_need));
            return PB_ERR_CAPACITY;
        }
        PB_TRY(upload(S->track_reg, S->h_track_reg.data(), sizeof(int64_t) * 2 * nr, st));
        e->track = S->d_track; e->track_reg = S->track_reg.as<int64_t>();
    }
    PB_CUDA(cudaEventRecord(E[0], st));
    int rc = pb_variant_encode_device(e, &V.d, V.d_regions, (int64_t) V.h_regions.size(), V.h_regions.data(), V.d_ref, 0, &S->params, room,
                                      e->p_images.as<int8_t>() + done * 33 * 26, e->p_positions.as<int64_t>() + done,
                                      e->p_depths.as<uint8_t>() + done, e->p_freqs.as<uint8_t>() + done,
                                      e->p_keys.as<char>() + done * PB_ALLELE_STRIDE, e->p_region_of.as<int32_t>() + done, nullptr, &n_g, (void *) st);
    e->track = nullptr; e->track_reg = nullptr;
    V.owned_end.clear();
    S->staged[b] = false; S->next_run = b ^ 1;
    if (rc == PB_OK) S->track_done += track_need;
    if (n_total) *n_total = done + n_g;
    if (rc != PB_OK) { if (rc == PB_ERR_CAPACITY) cudaStreamSynchronize(e->copy_stream); return rc; }
    for (int i = 0; i < 5; i++) S->enc_phase_ms[i] += e->ms[i];
    S->enc_launches += e->launches;
    if (n_g > 0 && S->region_id0[b] != 0)
        k_add_offset_i32<<<(unsigned) ceil_div(n_g, 256), 256, 0, st>>>(e->p_region_of.as<int32_t>() + done, n_g, S->region_id0[b]);
    PB_CUDA(cudaEventRecord(E[1], st));
    S->done = done + n_g;
    const int64_t avail = S->done - S->net_done;
    PB_TRY(stream_network(e, net, S, flush ? avail : avail / PIPE_NET_CHUNK * PIPE_NET_CHUNK));
    PB_CUDA(cudaEventRecord(E[2], st));
    S->groups++;
    return PB_OK;
}

extern "C" int pb_variant_stream_sync(pb_variant_encoder_t *e) {
    VariantStream *S;
    PB_TRY(session(e, &S, true));
    PB_CUDA(cudaStreamSynchronize(S->st));
    stream_collect_timing(S);
    return PB_OK;
}

// network over whatever is still waiting, wait for everything; *n_out = candidates of the session
extern "C" int pb_variant_stream_end(pb_variant_encoder_t *e, pb_variant_net_t *net, int64_t *n_out) {
    VariantStream *S;
    PB_TRY(session(e, &S, true));
    if (!net || !n_out) { set_error("null argument"); return PB_ERR_ARG; }
    cudaStream_t st = S->st;
    PB_CUDA(cudaStreamSynchronize(st));
    stream_collect_timing(S);
    if (S->done > S->net_done) {
        PB_CUDA(cudaEventRecord(e->pevt[1], st));
        PB_TRY(stream_network(e, net, S, S->done - S->net_done));
        PB_CUDA(cudaEventRecord(e->pevt[2], st));
        PB_CUDA(cudaStreamSynchronize(st));
        float b = 0.f;
        cudaEventElapsedTime(&b, e->pevt[1], e->pevt[2]);
        S->net_ms += b;
    }
    PB_CUDA(cudaStreamSynchronize(e->copy_stream));
    e->pms[0] = S->enc_ms; e->pms[1] = S->net_ms;
    *n_out = S->done;
    S->active = false;
    return PB_OK;
}

// per-phase encoder device time (ms: prefix, count, sites, alleles, windows) and kernel launches (encoder, network) of the
// last session, summed over its groups
extern "C" int pb_variant_stream_stats(pb_variant_encoder_t *e, float *ms5, int64_t *launches2, int64_t *groups) {
    if (!e || !e->vstream) { set_error("no session"); return PB_ERR_STATE; }
    VariantStream *S = e->vstream;
    if (ms5) for (int i = 0; i < 5; i++) ms5[i] = S->enc_phase_ms[i];
    if (launches2) { launches2[0] = S->enc_launches; launches2[1] = S->net_launches; }
    if (groups) *groups = S->groups;
    return PB_OK;
}

// device pointers of the session's accumulated columns and probabilities (valid until the next session begins)
extern "C" int pb_variant_stream_columns(pb_variant_encoder_t *e, pb_candidate_columns_t *cols, const float **d_probs, const int8_t **d_images) {
    if (!e || !cols) { set_error("null argument"); return PB_ERR_ARG; }
    cols->positions = e->p_positions.as<int64_t>(); cols->region_of = e->p_region_of.as<int32_t>();
    cols->depths = e->p_depths.as<uint8_t>(); cols->freqs = e->p_freqs.as<uint8_t>(); cols->keys = e->p_keys.as<char>();
    if (d_probs) *d_probs = e->p_probs.as<float>();
    if (d_images) *d_images = e->p_images.as<int8_t>();
    return PB_OK;
}

// D2H of the first n candidates of the last session (any pointer may be NULL)
extern "C" int pb_variant_stream_fetch(pb_variant_encoder_t *e, int64_t n, int8_t *h_images, int64_t *h_positions, uint8_t *h_depths,
                                       uint8_t *h_freqs, char *h_keys, int32_t *h_region_of, float *h_probs, void *stream_) {
    if (!e) { set_error("null handle"); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    if (n > 0) {
        if (h_images) PB_CUDA(cudaMemcpyAsync(h_images, e->p_images.p, (size_t) n * 33 * 26, cudaMemcpyDeviceToHost, st));
        if (h_positions) PB_CUDA(cudaMemcpyAsync(h_positions, e->p_positions.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, st));
        if (h_depths) PB_CUDA(cudaMemcpyAsync(h_depths, e->p_depths.p, n, cudaMemcpyDeviceToHost, st));
        if (h_freqs) PB_CUDA(cudaMemcpyAsync(h_freqs, e->p_freqs.p, n, cudaMemcpyDeviceToHost, st));
        if (h_keys) PB_CUDA(cudaMemcpyAsync(h_keys, e->p_keys.p, (size_t) n * PB_ALLELE_STRIDE, cudaMemcpyDeviceToHost, st));
        if (h_region_of) PB_CUDA(cudaMemcpyAsync(h_region_of, e->p_region_of.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
        if (h_probs) PB_CUDA(cudaMemcpyAsync(h_probs, e->p_probs.p, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, st));
    }
    PB_CUDA(cudaStreamSynchronize(st));
    return PB_OK;
}

// Host entry: regions are processed in groups; the H2D copy of group g+1 (copy stream, pinned source) overlaps the
// encoder + network kernels of group g, so PCIe time hides behind compute for all but the first group.
extern "C" int pb_variant_call_host(pb_variant_encoder_t *e, pb_variant_net_t *net, const pb_reads_t *h_reads,
                                    const pb_region_t *h_regions, int64_t n_regions, const char *h_ref, int64_t ref_bytes,
                                    const pb_variant_params_t *params, int64_t capacity, int8_t *h_images,
                                    int64_t *h_positions, uint8_t *h_depths, uint8_t *h_freqs, char *h_keys,
                                    int32_t *h_region_of, float *h_probs, int64_t *n_out, void *stream_) {
    if (!e || !net || !h_reads || !h_regions || !params || !n_out) { set_error("null argument"); return PB_ERR_ARG; }
    PB_CUDA(cudaSetDevice(e->device));
    *n_out = 0;
    if (n_regions <= 0) return PB_OK;
    bool ascending = true;
    for (int64_t r = 0; r < n_regions; r++) {
        if (h_regions[r].read_begin < 0 || h_regions[r].read_end > h_reads->n_reads || h_regions[r].read_begin > h_regions[r].read_end) {
            set_error("region %lld: read range out of bounds", (long long) r);
            return PB_ERR_ARG;
        }
        if (r > 0 && h_regions[r].read_begin < h_regions[r - 1].read_end) ascending = false;
    }
    if (n_regions <= CALL_GROUP || !ascending)
        return variant_call_host_single(e, net, h_reads, h_regions, n_regions, h_ref, ref_bytes, params, capacity, h_images, h_positions,
                                        h_depths, h_freqs, h_keys, h_region_of, h_probs, n_out, stream_);
    // group boundaries: a short first group keeps the un-overlapped first copy small
    std::vector<int64_t> gb;
    gb.push_back(0);
    for (int64_t r = std::min<int64_t>(CALL_FIRST_GROUP, n_regions); r < n_regions; r += CALL_GROUP) gb.push_back(r);
    gb.push_back(n_regions);
    const int64_t n_groups = (int64_t) gb.size() - 1;
    PB_TRY(pb_variant_stream_begin(e, net, params, capacity, nullptr, stream_));
    PB_TRY(pb_variant_stream_stage_host(e, h_reads, h_regions, gb[0], gb[1], h_ref, 0));
    for (int64_t g = 0; g < n_groups; g++) {
        int64_t n_tot = 0;
        const int rc = pb_variant_stream_run(e, net, g + 1 == n_groups, &n_tot);
        if (rc == PB_ERR_CAPACITY) {
            // the caller retries with the returned size: extrapolate from the regions seen so far (retried again if short)
            const int64_t need = (int64_t) ((double) n_tot * (double) n_regions / (double) gb[g + 1] * 1.25) + 4096;
            e->vstream->active = false;
            *n_out = need;
            set_error("candidate capacity %lld too small (estimated need %lld)", (long long) capacity, (long long) need);
            return PB_ERR_CAPACITY;
        }
        if (rc != PB_OK) { e->vstream->active = false; return rc; }
        // the network of this group is queued: issue the next group's copies now, so that neither the host work of staging nor
        // the copies themselves leave the compute stream idle
        // no sync here: the next run() builds its host-side tables while this group's network runs, and its encoder synchronises the
        // stream before any staging buffer is reused
        if (g + 1 < n_groups) PB_TRY(pb_variant_stream_stage_host(e, h_reads, h_regions, gb[g + 1], gb[g + 2], h_ref, (int32_t) gb[g + 1]));
    }
    PB_TRY(pb_variant_stream_end(e, net, n_out));
    return pb_variant_stream_fetch(e, *n_out, h_images, h_positions, h_depths, h_freqs, h_keys, h_region_of, h_probs, stream_);
}

extern "C" int pb_variant_call_timings(pb_variant_encoder_t *e, float *ms2) {
    if (!e || !ms2) return PB_ERR_ARG;
    ms2[0] = e->pms[0]; ms2[1] = e->pms[1];
    return PB_OK;
}

// Encodes regions [0, n_regions) into the encoder's column scratch (p_image / p_pos / p_idx) and cuts each region's columns into
// 1000-column images with 50 columns of overlap (AlignmentSummarizer.chunk_images): the image rows, in region then chunk order,
// with region ids counted from `region0`.  Synchronises `st` (the rows are planned on the host from the column offsets).
// *n_cols (optional): the encoded columns.
static int polish_encode_rows(pb_polish_encoder_t *e, const pb_reads_t *d_reads, const pb_region_t *d_regions, int64_t n_regions,
                              const pb_region_t *h_regions, int32_t region0, cudaStream_t st, std::vector<ChunkRow> &rows, int64_t *n_cols_out) {
    rows.clear();
    // encode into library scratch; column capacity: positions + generous insert allowance, retried on demand
    int64_t span = 0;
    for (int64_t r = 0; r < n_regions; r++) span += h_regions[r].ref_end - h_regions[r].ref_start + 1;
    int64_t cap_cols = 2 * span + 1024, n_cols = 0;
    for (int attempt = 0; attempt < 2; attempt++) {
        PB_TRY(e->p_image.reserve((size_t) cap_cols * 10));
        PB_TRY(e->p_pos.reserve(sizeof(int64_t) * cap_cols));
        PB_TRY(e->p_idx.reserve(sizeof(int32_t) * cap_cols));
        PB_TRY(e->p_col_off.reserve(sizeof(int64_t) * (n_regions + 1)));
        int rc = pb_polish_encode_device(e, d_reads, d_regions, n_regions, h_regions, cap_cols, e->p_image.as<uint8_t>(),
                                         e->p_pos.as<int64_t>(), e->p_idx.as<int32_t>(), e->p_col_off.as<int64_t>(), &n_cols, (void *) st);
        if (rc == PB_ERR_CAPACITY && attempt == 0) { cap_cols = n_cols + 16; continue; }
        if (rc != PB_OK) return rc;
        break;
    }
    if (n_cols_out) *n_cols_out = n_cols;
    std::vector<int64_t> col_off((size_t) n_regions + 1, 0);
    if (n_regions > 0) PB_CUDA(cudaMemcpyAsync(col_off.data(), e->p_col_off.p, sizeof(int64_t) * (n_regions + 1), cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    for (int64_t r = 0; r < n_regions; r++) {
        const int64_t n = col_off[r + 1] - col_off[r];
        int64_t start = 0, end = std::min<int64_t>(n, PB_POLISH_SEQ_LEN);
        int cid = 0;
        while (true) {
            ChunkRow c; c.col_start = col_off[r] + start; c.nvalid = (int32_t) (end - start); c.region = region0 + (int32_t) r; c.chunk_id = cid++; c.pad = 0;
            rows.push_back(c);
            if (end == n) break;
            start = end - 50;                                                  // SEQ_OVERLAP
            end = std::min<int64_t>(n, start + PB_POLISH_SEQ_LEN);
        }
    }
    return PB_OK;
}

extern "C" int pb_polish_call_device(pb_polish_encoder_t *e, pb_polish_net_t *net, const pb_reads_t *d_reads,
                                     const pb_region_t *d_regions, int64_t n_regions, const pb_region_t *h_regions,
                                     int64_t capacity_images, uint8_t *d_bases, uint8_t *d_phred, int64_t *d_position,
                                     int32_t *d_index, int32_t *d_image_region, int32_t *d_chunk_id, int64_t *n_images_out,
                                     void *stream_) {
    if (!e || !net || !n_images_out) { set_error("null argument"); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    PB_TRY(ensure_events(e->pevt, 3));
    PB_CUDA(cudaEventRecord(e->pevt[0], st));
    *n_images_out = 0;
    std::vector<ChunkRow> rows;
    PB_TRY(polish_encode_rows(e, d_reads, d_regions, n_regions, h_regions, 0, st, rows, nullptr));
    const int64_t n_img = (int64_t) rows.size();
    *n_images_out = n_img;
    if (n_img > capacity_images) {
        set_error("image capacity %lld < %lld needed", (long long) capacity_images, (long long) n_img);
        return PB_ERR_CAPACITY;
    }
    if (n_img > 0) {
        PB_TRY(upload(e->p_chunks, rows.data(), sizeof(ChunkRow) * n_img, st));
        PB_TRY(e->p_imgs.reserve((size_t) n_img * PB_POLISH_SEQ_LEN * PB_POLISH_FEATURES));
        k_polish_chunk<<<(unsigned) n_img, 256, 0, st>>>(e->p_chunks.as<ChunkRow>(), e->p_image.as<uint8_t>(), e->p_pos.as<int64_t>(),
                                                        e->p_idx.as<int32_t>(), e->p_imgs.as<uint8_t>(), d_position, d_index,
                                                        d_image_region, d_chunk_id);
        PB_CUDA(cudaGetLastError());
    }
    PB_CUDA(cudaEventRecord(e->pevt[1], st));
    if (n_img > 0) PB_TRY(pb_polish_net_forward_device(net, e->p_imgs.as<uint8_t>(), n_img, d_bases, d_phred, nullptr, nullptr, stream_));
    PB_CUDA(cudaEventRecord(e->pevt[2], st));
    PB_CUDA(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&e->pms[0], e->pevt[0], e->pevt[1]);
    cudaEventElapsedTime(&e->pms[1], e->pevt[1], e->pevt[2]);
    return PB_OK;
}

extern "C" int pb_polish_call_host(pb_polish_encoder_t *e, pb_polish_net_t *net, const pb_reads_t *h_reads,
                                   const pb_region_t *h_regions, int64_t n_regions, int64_t capacity_images, uint8_t *h_bases,
                                   uint8_t *h_phred, int64_t *h_position, int32_t *h_index, int32_t *h_image_region,
                                   int32_t *h_chunk_id, int64_t *n_images_out, void *stream_) {
    if (!e || !net || !h_reads || !h_regions || !n_images_out) { set_error("null argument"); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    PB_CUDA(cudaSetDevice(e->device));
    DevBuf *rb[8] = {&e->h_pos, &e->h_seq_off, &e->h_cigar_off, &e->h_flags, &e->h_mapq, &e->h_seq, &e->h_qual, &e->h_cigar};
    pb_reads_t d;
    PB_TRY(upload_reads(h_reads, rb, &d, st));
    PB_TRY(upload(e->h_regions, h_regions, sizeof(pb_region_t) * n_regions, st));
    const int64_t cap = std::max<int64_t>(capacity_images, 1);
    PB_TRY(e->p_bases.reserve((size_t) cap * PB_POLISH_SEQ_LEN));
    PB_TRY(e->p_phred.reserve((size_t) cap * PB_POLISH_SEQ_LEN));
    PB_TRY(e->p_position.reserve(sizeof(int64_t) * cap * PB_POLISH_SEQ_LEN));
    PB_TRY(e->p_index.reserve(sizeof(int32_t) * cap * PB_POLISH_SEQ_LEN));
    PB_TRY(e->p_iregion.reserve(sizeof(int32_t) * cap));
    PB_TRY(e->p_cid.reserve(sizeof(int32_t) * cap));
    PB_TRY(pb_polish_call_device(e, net, &d, e->h_regions.as<pb_region_t>(), n_regions, h_regions, capacity_images,
                                 e->p_bases.as<uint8_t>(), e->p_phred.as<uint8_t>(), e->p_position.as<int64_t>(),
                                 e->p_index.as<int32_t>(), e->p_iregion.as<int32_t>(), e->p_cid.as<int32_t>(), n_images_out, stream_));
    const int64_t n = *n_images_out;
    if (n > 0) {
        PB_CUDA(cudaMemcpyAsync(h_bases, e->p_bases.p, (size_t) n * PB_POLISH_SEQ_LEN, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_phred, e->p_phred.p, (size_t) n * PB_POLISH_SEQ_LEN, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_position, e->p_position.p, sizeof(int64_t) * n * PB_POLISH_SEQ_LEN, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_index, e->p_index.p, sizeof(int32_t) * n * PB_POLISH_SEQ_LEN, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_image_region, e->p_iregion.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
        PB_CUDA(cudaMemcpyAsync(h_chunk_id, e->p_cid.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    }
    PB_CUDA(cudaStreamSynchronize(st));
    return PB_OK;
}

extern "C" int pb_polish_call_timings(pb_polish_encoder_t *e, float *ms2) {
    if (!e || !ms2) return PB_ERR_ARG;
    ms2[0] = e->pms[0]; ms2[1] = e->pms[1];
    return PB_OK;
}

// ------------------------------------------------------------------------------------------- streaming polish session
// The polish counterpart of the variant session: groups of whole regions are staged and run one after the other; their images
// queue behind the ones still waiting for the network, the network runs over whole 8,192-image chunks as they fill, and after
// each network call the stitch-to-sink kernel appends that chunk's surviving bases to a caller-given device byte buffer at a
// running offset that never leaves the device.  Because a region never spans two groups, each group's consensus is the
// concatenation of its images' survivors, so the host only has to place the groups (the session counts bytes per group).
static constexpr int64_t POLISH_NET_CHUNK = 8192;          // POLISH_CHUNK of nets.cu

namespace pb {
struct PolishStream {
    bool active = false;
    cudaStream_t st = nullptr;
    char *d_sink = nullptr;
    int64_t capacity = 0;                       // sink records
    bool qualities = false;                     // records are (base, QV byte) pairs
    pb_edit_event_t *d_events = nullptr;        // edits session: the event sink (pb_polish_stream_edits)
    int64_t ev_capacity = 0;
    GroupView V[2];
    int32_t region_id0[2] = {0, 0};
    bool staged[2] = {false, false};
    int next_stage = 0, next_run = 0;
    // images encoded but not yet through the network; they are moved to the front of the buffers after every network call, so
    // fewer than one network chunk stays behind and the buffers hold at most one chunk plus one group's images
    int64_t pending = 0, ring_cap = 0;
    std::vector<int32_t> h_region, h_cid;       // host copy of the pending images' region id / chunk id
    int32_t prev_region = -1, prev_cid = 0;     // the last image that went through the network
    DevBuf imgs, position, index, region, cid, start, slot, draft;
    DevBuf bases, phred, counts, offsets, state, group_bytes, group_events, ev_scratch[2];
    int64_t group_cap = 0;
    std::vector<cudaEvent_t> ev;                // per group: encoder start, encoder end, network (+ sink) end
    int64_t ev_done = 0;
    float enc_ms = 0.f, net_ms = 0.f;
    int64_t cols = 0, images = 0, net_launches = 0, groups = 0;
};

void polish_stream_free(PolishStream *S) {
    if (!S) return;
    DevBuf *bufs[] = {&S->imgs, &S->position, &S->index, &S->region, &S->cid, &S->start, &S->slot, &S->draft, &S->bases, &S->phred,
                      &S->counts, &S->offsets, &S->state, &S->group_bytes, &S->group_events, &S->ev_scratch[0], &S->ev_scratch[1]};
    for (auto *b : bufs) b->release();
    for (auto x : S->ev) cudaEventDestroy(x);
    delete S;
}
}  // namespace pb

// grows `b` to `need` bytes keeping its first `keep` bytes
static int grow_keep(DevBuf &b, size_t need, size_t keep, cudaStream_t st) {
    if (need <= b.cap) return PB_OK;
    DevBuf n;
    PB_TRY(n.reserve(need));
    if (keep) PB_CUDA(cudaMemcpyAsync(n.p, b.p, keep, cudaMemcpyDeviceToDevice, st));
    PB_CUDA(cudaStreamSynchronize(st));
    b.release();
    b = n;
    return PB_OK;
}

// bytes per pending image in each image buffer (images, position, index, region, chunk id, region start, group slot, and in an
// edits session the columns' draft bases)
static const size_t PS_BYTES[8] = {(size_t) PB_POLISH_SEQ_LEN * PB_POLISH_FEATURES, sizeof(int64_t) * PB_POLISH_SEQ_LEN,
                                   sizeof(int32_t) * PB_POLISH_SEQ_LEN, sizeof(int32_t), sizeof(int32_t), sizeof(int64_t), sizeof(int32_t),
                                   (size_t) PB_POLISH_SEQ_LEN};
// the image buffers of the session; returns how many are in use
static int ps_buffers(PolishStream *S, DevBuf *B[8]) {
    B[0] = &S->imgs; B[1] = &S->position; B[2] = &S->index; B[3] = &S->region; B[4] = &S->cid; B[5] = &S->start; B[6] = &S->slot;
    B[7] = &S->draft;
    return S->d_events ? 8 : 7;
}

static int psession(pb_polish_encoder_t *e, PolishStream **S, bool need_active) {
    if (!e) { set_error("null handle"); return PB_ERR_ARG; }
    if (!e->pstream) e->pstream = new PolishStream();
    *S = e->pstream;
    if (need_active && !(*S)->active) { set_error("no active stream session: call pb_polish_stream_begin first"); return PB_ERR_STATE; }
    return PB_OK;
}

static int polish_stream_begin(pb_polish_encoder_t *e, pb_polish_net_t *net, int64_t capacity, char *d_sink, bool qualities, void *stream_) {
    if (!e || !net || (capacity > 0 && !d_sink)) { set_error("null argument"); return PB_ERR_ARG; }
    PolishStream *S;
    PB_TRY(psession(e, &S, false));
    PB_CUDA(cudaSetDevice(e->device));
    if (!e->copy_stream) {
        PB_CUDA(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
        for (int b = 0; b < 2; b++) PB_CUDA(cudaEventCreateWithFlags(&e->copied[b], cudaEventDisableTiming));
    }
    PB_TRY(ensure_events(e->pevt, 3));
    S->st = (cudaStream_t) stream_;
    S->d_sink = d_sink; S->capacity = std::max<int64_t>(capacity, 0); S->qualities = qualities;
    S->d_events = nullptr; S->ev_capacity = 0;
    S->staged[0] = S->staged[1] = false; S->next_stage = 0; S->next_run = 0;
    S->pending = 0; S->h_region.clear(); S->h_cid.clear(); S->prev_region = -1; S->prev_cid = 0;
    S->ev_done = 0; S->enc_ms = S->net_ms = 0.f;
    S->cols = S->images = S->net_launches = S->groups = 0;
    PB_TRY(S->state.reserve(2 * sizeof(int64_t)));
    if (S->group_cap == 0) { PB_TRY(S->group_bytes.reserve(sizeof(int64_t) * 256)); S->group_cap = 256; }
    PB_CUDA(cudaMemsetAsync(S->state.p, 0, 2 * sizeof(int64_t), S->st));
    PB_CUDA(cudaMemsetAsync(S->group_bytes.p, 0, sizeof(int64_t) * S->group_cap, S->st));
    S->active = true;
    return PB_OK;
}

extern "C" int pb_polish_stream_begin(pb_polish_encoder_t *e, pb_polish_net_t *net, int64_t capacity_bytes, char *d_sink, void *stream_) {
    return polish_stream_begin(e, net, capacity_bytes, d_sink, false, stream_);
}

// the same session with a sink of 2-byte (base, QV byte) records: d_sink holds 2 * capacity_records bytes
extern "C" int pb_polish_stream_begin_qual(pb_polish_encoder_t *e, pb_polish_net_t *net, int64_t capacity_records, char *d_sink,
                                           void *stream_) {
    return polish_stream_begin(e, net, capacity_records, d_sink, true, stream_);
}

// the event sink of an edits session: set after _begin, before the first group is staged
extern "C" int pb_polish_stream_edits(pb_polish_encoder_t *e, int64_t capacity_events, pb_edit_event_t *d_events) {
    PolishStream *S;
    PB_TRY(psession(e, &S, true));
    if (!d_events) { set_error("null argument"); return PB_ERR_ARG; }
    if (S->groups > 0 || S->staged[0] || S->staged[1]) { set_error("the event sink is attached before the first stage"); return PB_ERR_STATE; }
    S->d_events = d_events; S->ev_capacity = std::max<int64_t>(capacity_events, 0);
    if (S->ring_cap > 0) PB_TRY(S->draft.reserve(PS_BYTES[7] * S->ring_cap));      // the ring may have grown in an earlier session
    if (S->group_events.cap < sizeof(int64_t) * S->group_cap) PB_TRY(S->group_events.reserve(sizeof(int64_t) * S->group_cap));
    PB_CUDA(cudaMemsetAsync(S->group_events.p, 0, sizeof(int64_t) * S->group_cap, S->st));
    return PB_OK;
}

// regions [g0, g1) of a workload resident in HBM: only the re-based region rows are copied (copy stream).  d_ref: the group's
// reference strings (an edits session reads each column's draft base from them when the group is run)
static int polish_stream_stage(pb_polish_encoder_t *e, const pb_reads_t *d_reads, const pb_region_t *h_regions, int64_t g0, int64_t g1,
                               int32_t region_id0, const char *d_ref) {
    PolishStream *S;
    PB_TRY(psession(e, &S, true));
    if (S->d_events && !d_ref) { set_error("an edits session stages groups with their reference (_stage_device_draft)"); return PB_ERR_ARG; }
    if (!d_reads || !h_regions || g0 < 0 || g1 <= g0) { set_error("bad group [%lld, %lld)", (long long) g0, (long long) g1); return PB_ERR_ARG; }
    const int b = S->next_stage;
    if (S->staged[b]) { set_error("both staging buffers are in use: run a staged group first"); return PB_ERR_STATE; }
    GroupView &V = S->V[b];
    const int64_t r0 = h_regions[g0].read_begin, r1 = h_regions[g1 - 1].read_end;
    if (r0 < 0 || r1 > d_reads->n_reads || r1 < r0) { set_error("group read range out of bounds"); return PB_ERR_ARG; }
    V.h_regions.assign(h_regions + g0, h_regions + g1);
    for (auto &rg : V.h_regions) { rg.read_begin -= r0; rg.read_end -= r0; }
    PB_TRY(upload(e->g_regions[b], V.h_regions.data(), sizeof(pb_region_t) * V.h_regions.size(), e->copy_stream));
    PB_CUDA(cudaEventRecord(e->copied[b], e->copy_stream));
    V.d = *d_reads;
    V.d.n_reads = r1 - r0;
    V.d.pos += r0; V.d.seq_off += r0; V.d.cigar_off += r0; V.d.flags += r0; V.d.mapq += r0;     // seq / qual / cigar keep absolute offsets
    V.d_regions = e->g_regions[b].as<pb_region_t>();
    V.d_ref = d_ref;
    S->staged[b] = true; S->region_id0[b] = region_id0; S->next_stage = b ^ 1;
    return PB_OK;
}

extern "C" int pb_polish_stream_stage_device(pb_polish_encoder_t *e, const pb_reads_t *d_reads, const pb_region_t *h_regions,
                                             int64_t g0, int64_t g1, int32_t region_id0) {
    return polish_stream_stage(e, d_reads, h_regions, g0, g1, region_id0, nullptr);
}

extern "C" int pb_polish_stream_stage_device_draft(pb_polish_encoder_t *e, const pb_reads_t *d_reads, const pb_region_t *h_regions,
                                                   int64_t g0, int64_t g1, int32_t region_id0, const char *d_ref) {
    if (!d_ref) { set_error("null reference"); return PB_ERR_ARG; }
    return polish_stream_stage(e, d_reads, h_regions, g0, g1, region_id0, d_ref);
}

// the network + stitch-to-sink over every whole chunk of the pending images (`flush`: over all of them), then the images left
// behind move to the front of the buffers
static int polish_stream_network(pb_polish_net_t *net, PolishStream *S, bool flush) {
    cudaStream_t st = S->st;
    int64_t done = 0;
    while (true) {
        const int64_t left = S->pending - done, B = std::min(left, POLISH_NET_CHUNK);
        if (B <= 0 || (!flush && left < POLISH_NET_CHUNK)) break;
        PB_TRY(S->bases.reserve((size_t) POLISH_NET_CHUNK * PB_POLISH_SEQ_LEN));
        PB_TRY(S->phred.reserve((size_t) POLISH_NET_CHUNK * PB_POLISH_SEQ_LEN));
        PB_TRY(pb_polish_net_forward_device(net, S->imgs.as<uint8_t>() + done * PS_BYTES[0], B, S->bases.as<uint8_t>(), S->phred.as<uint8_t>(),
                                            nullptr, nullptr, (void *) st));
        int64_t nl = 0;
        pb_polish_net_launches(net, &nl);
        S->net_launches += nl;
        SinkArgs A;
        A.bases = S->bases.as<uint8_t>();
        A.phred = S->qualities ? S->phred.as<uint8_t>() : nullptr;
        A.position = S->position.as<int64_t>() + done * PB_POLISH_SEQ_LEN; A.index = S->index.as<int32_t>() + done * PB_POLISH_SEQ_LEN;
        A.region = S->region.as<int32_t>() + done; A.cid = S->cid.as<int32_t>() + done;
        A.start = S->start.as<int64_t>() + done; A.slot = S->slot.as<int32_t>() + done;
        A.n = B; A.n_known = S->pending - done;
        A.prev_region = done > 0 ? S->h_region[done - 1] : S->prev_region;
        A.prev_cid = done > 0 ? S->h_cid[done - 1] : S->prev_cid;
        A.state = S->state.as<int64_t>(); A.group_bytes = S->group_bytes.as<int64_t>(); A.out = S->d_sink; A.capacity = S->capacity;
        if (S->d_events) {
            A.edit_phred = S->phred.as<uint8_t>(); A.draft = S->draft.as<uint8_t>() + done * PB_POLISH_SEQ_LEN;
            A.events = S->d_events; A.ev_capacity = S->ev_capacity; A.group_events = S->group_events.as<int64_t>();
        }
        PB_TRY(polish_sink(A, S->counts, S->offsets, st, S->ev_scratch));
        done += B;
    }
    if (done == 0) return PB_OK;
    S->prev_region = S->h_region[done - 1]; S->prev_cid = S->h_cid[done - 1];
    const int64_t tail = S->pending - done;          // < one chunk <= done: source and destination do not overlap
    DevBuf *Bf[8];
    const int nb = ps_buffers(S, Bf);
    if (tail > 0)
        for (int k = 0; k < nb; k++)
            PB_CUDA(cudaMemcpyAsync(Bf[k]->p, Bf[k]->as<char>() + done * PS_BYTES[k], tail * PS_BYTES[k], cudaMemcpyDeviceToDevice, st));
    S->h_region.erase(S->h_region.begin(), S->h_region.begin() + done);
    S->h_cid.erase(S->h_cid.begin(), S->h_cid.begin() + done);
    S->pending = tail;
    return PB_OK;
}

// Encode the oldest staged group, queue its images behind the pending ones, and run the network + sink over the whole chunks
// available (`flush`: over everything).  Returns with the kernels still running.  *n_total = encoded columns of the session so
// far, an upper bound of its consensus bytes (each column survives at most once).
extern "C" int pb_polish_stream_run(pb_polish_encoder_t *e, pb_polish_net_t *net, int flush, int64_t *n_total) {
    PolishStream *S;
    PB_TRY(psession(e, &S, true));
    if (!net) { set_error("null handle"); return PB_ERR_ARG; }
    const int b = S->next_run;
    if (!S->staged[b]) { set_error("no staged group"); return PB_ERR_STATE; }
    cudaStream_t st = S->st;
    cudaEvent_t *E;
    PB_TRY(stream_events(S, S->groups, &E));
    PB_CUDA(cudaStreamWaitEvent(st, e->copied[b], 0));
    GroupView &V = S->V[b];
    const int32_t region0 = S->region_id0[b];
    PB_CUDA(cudaEventRecord(E[0], st));
    std::vector<ChunkRow> rows;
    int64_t n_cols = 0;
    const int rc = polish_encode_rows(e, &V.d, V.d_regions, (int64_t) V.h_regions.size(), V.h_regions.data(), region0, st, rows, &n_cols);
    S->staged[b] = false; S->next_run = b ^ 1;
    if (rc != PB_OK) return rc;
    const int64_t slot = S->groups, n_new = (int64_t) rows.size(), p0 = S->pending;
    if (slot >= S->group_cap) {
        const int64_t cap = 2 * S->group_cap;
        PB_TRY(grow_keep(S->group_bytes, sizeof(int64_t) * cap, sizeof(int64_t) * S->group_cap, st));
        PB_CUDA(cudaMemsetAsync(S->group_bytes.as<int64_t>() + S->group_cap, 0, sizeof(int64_t) * (cap - S->group_cap), st));
        if (S->d_events) {
            PB_TRY(grow_keep(S->group_events, sizeof(int64_t) * cap, sizeof(int64_t) * S->group_cap, st));
            PB_CUDA(cudaMemsetAsync(S->group_events.as<int64_t>() + S->group_cap, 0, sizeof(int64_t) * (cap - S->group_cap), st));
        }
        S->group_cap = cap;
    }
    if (p0 + n_new > S->ring_cap) {
        DevBuf *Bf[8];
        const int nb = ps_buffers(S, Bf);
        const int64_t cap = std::max<int64_t>(p0 + n_new, POLISH_NET_CHUNK);
        for (int k = 0; k < nb; k++) PB_TRY(grow_keep(*Bf[k], PS_BYTES[k] * cap, PS_BYTES[k] * p0, st));
        S->ring_cap = cap;
    }
    if (n_new > 0) {
        std::vector<int64_t> h_start((size_t) n_new);
        std::vector<int32_t> h_slot((size_t) n_new, (int32_t) slot);
        for (int64_t k = 0; k < n_new; k++) {
            h_start[k] = V.h_regions[rows[k].region - region0].ref_start;
            S->h_region.push_back(rows[k].region); S->h_cid.push_back(rows[k].chunk_id);
        }
        PB_TRY(upload(e->p_chunks, rows.data(), sizeof(ChunkRow) * n_new, st));
        k_polish_chunk<<<(unsigned) n_new, 256, 0, st>>>(e->p_chunks.as<ChunkRow>(), e->p_image.as<uint8_t>(), e->p_pos.as<int64_t>(),
                                                         e->p_idx.as<int32_t>(), S->imgs.as<uint8_t>() + p0 * PS_BYTES[0],
                                                         S->position.as<int64_t>() + p0 * PB_POLISH_SEQ_LEN,
                                                         S->index.as<int32_t>() + p0 * PB_POLISH_SEQ_LEN, S->region.as<int32_t>() + p0,
                                                         S->cid.as<int32_t>() + p0,
                                                         S->d_events ? S->draft.as<uint8_t>() + p0 * PB_POLISH_SEQ_LEN : nullptr,
                                                         V.d_ref, V.d_regions, region0);
        PB_CUDA(cudaGetLastError());
        PB_CUDA(cudaMemcpyAsync(S->start.as<int64_t>() + p0, h_start.data(), sizeof(int64_t) * n_new, cudaMemcpyHostToDevice, st));
        PB_CUDA(cudaMemcpyAsync(S->slot.as<int32_t>() + p0, h_slot.data(), sizeof(int32_t) * n_new, cudaMemcpyHostToDevice, st));
    }
    S->pending = p0 + n_new;
    S->cols += n_cols; S->images += n_new;
    PB_CUDA(cudaEventRecord(E[1], st));
    PB_TRY(polish_stream_network(net, S, flush != 0));
    PB_CUDA(cudaEventRecord(E[2], st));
    S->groups++;
    if (n_total) *n_total = S->cols;
    return PB_OK;
}

extern "C" int pb_polish_stream_sync(pb_polish_encoder_t *e) {
    PolishStream *S;
    PB_TRY(psession(e, &S, true));
    PB_CUDA(cudaStreamSynchronize(S->st));
    stream_collect_timing(S);
    return PB_OK;
}

// network + sink over whatever is still pending, wait for everything; *n_out = consensus records of the session (bytes, or
// (base, QV byte) pairs in a _begin_qual session).  PB_ERR_CAPACITY: the sink was too small, *n_out = the records it needed (the
// records past the capacity were not written: restart larger).
extern "C" int pb_polish_stream_end(pb_polish_encoder_t *e, pb_polish_net_t *net, int64_t *n_out) {
    PolishStream *S;
    PB_TRY(psession(e, &S, true));
    if (!net || !n_out) { set_error("null argument"); return PB_ERR_ARG; }
    cudaStream_t st = S->st;
    S->active = false;
    PB_CUDA(cudaStreamSynchronize(st));
    stream_collect_timing(S);
    if (S->pending > 0) {
        PB_CUDA(cudaEventRecord(e->pevt[1], st));
        PB_TRY(polish_stream_network(net, S, true));
        PB_CUDA(cudaEventRecord(e->pevt[2], st));
        PB_CUDA(cudaStreamSynchronize(st));
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e->pevt[1], e->pevt[2]);
        S->net_ms += ms;
    }
    int64_t total = 0;
    PB_CUDA(cudaMemcpyAsync(&total, S->state.p, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    PB_CUDA(cudaStreamSynchronize(e->copy_stream));
    e->pms[0] = S->enc_ms; e->pms[1] = S->net_ms;
    *n_out = total;
    if (total > S->capacity) {
        set_error("consensus sink capacity %lld < %lld bytes needed", (long long) S->capacity, (long long) total);
        return PB_ERR_CAPACITY;
    }
    if (S->d_events) {
        int64_t n_ev = 0;
        PB_TRY(pb_polish_stream_event_total(e, &n_ev));
        if (n_ev > S->ev_capacity) {
            set_error("edit event sink capacity %lld < %lld events needed", (long long) S->ev_capacity, (long long) n_ev);
            return PB_ERR_CAPACITY;
        }
    }
    return PB_OK;
}

// events needed by the last edits session so far (all of them after _end)
extern "C" int pb_polish_stream_event_total(pb_polish_encoder_t *e, int64_t *n_events) {
    if (!e || !e->pstream || !e->pstream->d_events) { set_error("no edits session"); return PB_ERR_STATE; }
    if (!n_events) { set_error("null argument"); return PB_ERR_ARG; }
    PolishStream *S = e->pstream;
    PB_CUDA(cudaMemcpyAsync(n_events, S->state.as<int64_t>() + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, S->st));
    PB_CUDA(cudaStreamSynchronize(S->st));
    return PB_OK;
}

// events of each group of the last edits session, in the order the groups were run (call after _end)
extern "C" int pb_polish_stream_group_events(pb_polish_encoder_t *e, int64_t *h_events, int64_t n_groups) {
    if (!e || !e->pstream || !e->pstream->d_events) { set_error("no edits session"); return PB_ERR_STATE; }
    PolishStream *S = e->pstream;
    if (!h_events || n_groups < 0 || n_groups > S->groups) { set_error("bad argument"); return PB_ERR_ARG; }
    if (n_groups == 0) return PB_OK;
    PB_CUDA(cudaMemcpyAsync(h_events, S->group_events.p, sizeof(int64_t) * n_groups, cudaMemcpyDeviceToHost, S->st));
    PB_CUDA(cudaStreamSynchronize(S->st));
    return PB_OK;
}

// the last session: device ms [encoder, network + sink] summed over its groups; counts [groups, images, encoded columns,
// network launches]
extern "C" int pb_polish_stream_stats(pb_polish_encoder_t *e, float *ms2, int64_t *counts4) {
    if (!e || !e->pstream) { set_error("no session"); return PB_ERR_STATE; }
    PolishStream *S = e->pstream;
    if (ms2) { ms2[0] = S->enc_ms; ms2[1] = S->net_ms; }
    if (counts4) { counts4[0] = S->groups; counts4[1] = S->images; counts4[2] = S->cols; counts4[3] = S->net_launches; }
    return PB_OK;
}

// consensus bytes of each group of the last session, in the order the groups were run (call after _end)
extern "C" int pb_polish_stream_group_bytes(pb_polish_encoder_t *e, int64_t *h_bytes, int64_t n_groups) {
    if (!e || !e->pstream) { set_error("no session"); return PB_ERR_STATE; }
    PolishStream *S = e->pstream;
    if (!h_bytes || n_groups < 0 || n_groups > S->groups) { set_error("bad argument"); return PB_ERR_ARG; }
    if (n_groups == 0) return PB_OK;
    PB_CUDA(cudaMemcpyAsync(h_bytes, S->group_bytes.p, sizeof(int64_t) * n_groups, cudaMemcpyDeviceToHost, S->st));
    PB_CUDA(cudaStreamSynchronize(S->st));
    return PB_OK;
}
