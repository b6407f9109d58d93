// Opaque handle layouts shared by the translation units of libpepper_b200.
#pragma once
#include "common.cuh"
#include <vector>

namespace pb {
struct VariantStream;      // streaming session state (pipeline.cu)
// network layers (nets_tc.cu): weights as 16-bit hi/lo tile images + the fp32 bias; per-chunk tiled operands
// `scale`: the power of two s the tiles hold s W in (max |s W| in (2^14, 2^15]); the epilogues multiply by 1 / s
// wh_hi / wh_lo (the variant encoder only): the same weights in 128-row half tiles for k_lstm_layer_enc
struct TcRnn { DevBuf w_hi, w_lo, wh_hi, wh_lo, bias; int nkt_x = 0, nkt_h = 0; float scale = 1.f; };
struct TcLin { DevBuf w_hi, w_lo, bias; int nkt = 0; float scale = 1.f; };
// a weight matrix on int8 slices (mode 2: the decoder layer, tc_gemm.cuh k_lstm_layer_q8, and linear_1, k_gemm_q8): the two
// slices of round(sw_n W[n][k]), sw_n = 32512 / max_k |W[n][k]| over the row's K (the decoder: [W_ih | W_hh]), as
// [N / 128 n-tiles][K / 64 k-tiles][128][64] byte images, and the epilogue's 256 / (32512 sw_n) per output column n.  err: the
// largest weight-only estimate over the rows of the error the slices add to a pre-activation (nets_tc.cu tc_upload_q8);
// pb_variant_net_create compares it with PB_VARIANT_Q8_MAX_GATE_ERR (decoder) and PB_VARIANT_Q8_HEAD_MAX_ERR (linear_1)
struct TcQ8 { DevBuf w1, w0, col_scale; double err = 0.0; };
struct TcVariant {
    TcRnn enc[2], dec[2];
    TcLin lin[5];
    TcQ8 decq[2], lin1q;
    // mode 2: the encoder writes the decoder's x slices (q1 | q0) into yenc_lo, the decoder its own h slices into ydec_q, and
    // linear_1 reads those; ydec_hi / ydec_lo (the decoder's fp16 output) exist in mode 1 only
    DevBuf img_op, yenc_hi, yenc_lo, ydec_hi, ydec_lo, ydec_q, c, act_hi[2], act_lo[2], final_f32;
    // which GEMMs execute the third (a_lo x w_hi) product: bit 0 encoder h-part, 1 decoder x-part, 2 decoder h-part, 3 linear_1,
    // 4 linear_2..5; clearing a bit runs that GEMM with two products, 0x1f = three everywhere.  Default 0x1a: the recurrent
    // (h-part) GEMMs of both LSTM layers run with two products — each passes the parity gate on its own (hidden states within
    // 1e-3, class index exact outside the 1e-4 margin; DESIGN.md section 4 has the per-GEMM errors) — while the decoder's x-part
    // and the MLP head, which fail it, keep three.
    int lo_mask = 0x1a;
};
struct TcPolish {
    TcRnn enc[2], dec[2];
    DevBuf img_op, yenc_hi, yenc_lo, ydec_hi, ydec_lo, zero, flags;
    int lo_mask = 0x7;      // bit 0 encoder h-part, 1 decoder x-part, 2 decoder h-part
};
// optional record sink of the variant head kernel: the encoder's columns of the candidates of this forward call + output records
struct OutSink {
    pb_candidate_columns_t cols{nullptr, nullptr, nullptr, nullptr, nullptr};
    pb_pred_record_t *records = nullptr;
    OutSink at(int64_t b0) const {
        OutSink S = *this;
        if (records) {
            S.cols.positions += b0; S.cols.region_of += b0; S.cols.depths += b0; S.cols.freqs += b0; S.cols.keys += b0 * PB_ALLELE_STRIDE;
            S.records += b0;
        }
        return S;
    }
};
// one network chunk of polish predictions for the stitch-to-sink kernel (stitch.cu)
struct SinkArgs {
    const uint8_t *bases = nullptr;                              // [n][1000] network output of the chunk
    const uint8_t *phred = nullptr;                              // [n][1000] its phred; set: 2-byte (base, QV byte) records
    const int64_t *position = nullptr; const int32_t *index = nullptr;   // [n][1000]
    const int32_t *region = nullptr, *cid = nullptr;             // [n_known] image region / chunk id from the chunk's first image
    const int64_t *start = nullptr;                              // [n] start of each image's region
    const int32_t *slot = nullptr;                               // [n] group_bytes slot of each image
    int64_t n = 0, n_known = 0;
    int32_t prev_region = -1, prev_cid = 0;                      // the image before the chunk (region -1: none)
    int32_t *counts = nullptr; const int64_t *offsets = nullptr; // scratch (set by polish_sink)
    int64_t *state = nullptr;                                    // [0] running sink offset (records needed so far)
    int64_t *group_bytes = nullptr;                              // records per slot
    char *out = nullptr; int64_t capacity = 0;                   // capacity in records
    // edits session (events set): the columns' phred and draft bases [n][1000] and the event sink; state[1] = events needed
    // so far
    const uint8_t *edit_phred = nullptr, *draft = nullptr;
    pb_edit_event_t *events = nullptr; int64_t ev_capacity = 0;
    int64_t *group_events = nullptr;                             // events per slot
    int32_t *ev_counts = nullptr; const int64_t *ev_offsets = nullptr;   // scratch (set by polish_sink)
};
// ev: two scratch buffers (event counts, event offsets), needed when A.events is set
int polish_sink(SinkArgs A, DevBuf &counts, DevBuf &offsets, cudaStream_t st, DevBuf *ev = nullptr);
struct PolishStream;       // streaming polish session state (pipeline.cu)
void polish_stream_free(PolishStream *S);
int tc_upload_rnn(TcRnn &T, const float *Wp, const float *bias, int K0, int K0p_src, int H, int Kp_src, bool half_tiles = false);
int tc_upload_lin(TcLin &T, const float *w, const float *bias, int N, int K);
int tc_upload_rnn_q8(TcQ8 &T, const float *Wp, int K0, int K0p_src, int H, int Kp_src);
int tc_upload_q8(TcQ8 &T, const float *W, int N, int K, bool a_quant);
}  // namespace pb

struct pb_variant_encoder {
    int device = 0;
    pb::DevBuf op_ref, op_rd, read_reflen, read_region, tile_region, tile_x0, region_goff, M16, cov, meta, dbg,
        tile_nsites, tile_nev, tile_site_base, tile_ev_base, site_of, site_g, site_evoff, site_cur, ev, cand_tmp,
        site_ncand, site_region, site_candoff, rare, scalars;
    // host-entry staging
    pb::DevBuf h_pos, h_seq_off, h_cigar_off, h_flags, h_mapq, h_seq, h_qual, h_cigar, h_regions, h_ref;
    pb::DevBuf o_images, o_positions, o_depths, o_freqs, o_keys, o_region_of, o_per_region;
    cudaEvent_t evt[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    float ms[5] = {0, 0, 0, 0, 0};
    bool debug = false;
    // last-call bookkeeping for the debug read-back
    std::vector<int64_t> last_goff;
    std::vector<pb_region_t> last_regions;
    const char *last_d_ref = nullptr;
    size_t rare_cap = 1 << 20;
    // fused call scratch (pipeline.cu)
    pb::DevBuf p_images, p_positions, p_depths, p_freqs, p_keys, p_region_of, p_probs, p_per_region;
    cudaEvent_t pevt[3] = {nullptr, nullptr, nullptr};
    float pms[2] = {0, 0};
    int64_t launches = 0;
    // pipelined host entry (pipeline.cu): double-buffered staging + copy stream
    pb::DevBuf g_buf[2][10];
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t copied[2] = {nullptr, nullptr};
    pb::VariantStream *vstream = nullptr;
    // gVCF track of a streaming session (pb_variant_stream_track), set for the duration of one group's encode
    uint32_t *track = nullptr;
    const int64_t *track_reg = nullptr;
};

struct pb_polish_encoder {
    int device = 0;
    pb::DevBuf op_ref, op_rd, read_reflen, read_region, tile_region, tile_x0, region_goff, basecnt, cov, longest, tile_ncols,
        tile_col_base, col_of, inscnt, scalars;
    pb::DevBuf h_pos, h_seq_off, h_cigar_off, h_flags, h_mapq, h_seq, h_qual, h_cigar, h_regions;
    pb::DevBuf o_image, o_pos, o_idx, o_col_off;
    cudaEvent_t evt[4] = {nullptr, nullptr, nullptr, nullptr};
    float ms[3] = {0, 0, 0};
    // fused call scratch (pipeline.cu)
    pb::DevBuf p_image, p_pos, p_idx, p_col_off, p_chunks, p_imgs, p_position, p_index, p_bases, p_phred, p_iregion, p_cid;
    cudaEvent_t pevt[3] = {nullptr, nullptr, nullptr};
    float pms[2] = {0, 0};
    int64_t launches = 0;
    // streaming session (pipeline.cu): double-buffered region rows + copy stream
    pb::DevBuf g_regions[2];
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t copied[2] = {nullptr, nullptr};
    pb::PolishStream *pstream = nullptr;
};

struct pb_variant_net {
    int device = 0;
    // 1 = wgmma GEMMs on the fp16 hi/lo operand split, 2 = mode 1 with the decoder LSTM and linear_1 on int8 tensor cores.
    // pb_variant_net_create picks 2 when both pass the int8 guard (q8_gate_err < PB_VARIANT_Q8_MAX_GATE_ERR and
    // q8_head_err < PB_VARIANT_Q8_HEAD_MAX_ERR), else 1
    int mode = 2;
    double q8_gate_err = 0.0, q8_head_err = 0.0;
    pb::TcVariant tc;
    pb::DevBuf out_w, out_b;    // output_layer_type (3 x 512) for k_variant_out
    pb::DevBuf img, probs;      // host-entry staging
    int64_t launches = 0;
};

struct pb_polish_net {
    int device = 0;
    pb::TcPolish tc;
    pb::DevBuf dW, dB;          // dense1 (5 x 256) for k_polish_dense_tiles
    pb::DevBuf acc, img, bases, phred;
    int64_t launches = 0;
};

namespace pb {
int variant_forward_tc(pb_variant_net *N, const int8_t *d_images, int64_t B, float *d_probs, float *d_hidden_dbg, cudaStream_t st,
                       const OutSink &sink);
int polish_forward_tc(pb_polish_net *N, const uint8_t *d_images, int64_t B, int64_t n_total, int64_t b0, float *d_hidden_dbg,
                      cudaStream_t st);
}  // namespace pb
