// Recurrent-network inference for sm_90a, host side of both networks: the parameter tables, weight packing, handle lifetime
// and the forward entry points of the variant network (bi-LSTM x2 + MLP head) and the polish network (bi-GRU x2 + Linear with
// the 19-window sliding loop).  Every layer runs on the wgmma kernels of tc_gemm.cuh, launched one chunk at a time by
// nets_tc.cu; this file splits the input into chunks and turns the polish network's accumulated softmax into bases and phred.
//
// Packing: weight rows are re-ordered so that the 4 gate pre-activations of one hidden unit are adjacent rows 4j+g, with
// the input projection (W_ih) and the recurrent weights (W_hh) side by side in one K range; the GRU's n gate keeps its x-part
// and h-part in separate rows (n = tanh(W_in x + b_in + r * (W_hn h + b_hn)), pepper simple_model.py:12 -> torch.nn.GRU
// semantics).  nets_tc.cu tiles the packed rows for the tensor cores.
#include "handles.cuh"
#include <vector>
#include <algorithm>
#include <math.h>

namespace pb {

// the packed rows' K = [x | pad | h | pad] is padded to a multiple of PACK_KPAD (tc_upload_rnn / tc_upload_rnn_q8 read it at
// that stride)
constexpr int PACK_KPAD = 16;

// ------------------------------------------------------------------ polish head
// torch.max(acc, 2) (first maximal index) and phred = -10 log10(1 - v/count), inf -> 100,
// count = 2 on columns [50, 950) else 1 (predict_distributed_cpu.py:83-90); stored as uint8 (DataStorePredict.py:49)
__global__ void k_polish_finalize(const float *__restrict__ acc, uint8_t *__restrict__ bases, uint8_t *__restrict__ phred, int64_t n_img) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_img * 1000) return;
    const float *a = acc + i * 5;
    int best = 0; float bv = a[0];
#pragma unroll
    for (int c = 1; c < 5; c++) if (a[c] > bv) { bv = a[c]; best = c; }
    const int col = (int) (i % 1000);
    const float count = (col >= 50 && col < 950) ? 2.0f : 1.0f;
    float ph = -10.0f * log10f(1.0f - bv / count);
    if (isinf(ph)) ph = 100.0f;
    bases[i] = (uint8_t) best;
    // numpy astype(uint8) of a float: truncation toward zero (negative / NaN values are implementation defined there)
    phred[i] = (uint8_t) (int) fmaxf(0.f, fminf(ph, 255.f));
}

// ------------------------------------------------------------------ host helpers
static int round_up(int x, int m) { return (x + m - 1) / m * m; }

struct PackedRnn {      // one direction of one layer
    std::vector<float> W, bias;
    int K0, K0p, Kp;
};

// PyTorch LSTM params (gate order i,f,g,o) -> rows 4j+g, K = [x | pad | h | pad]
static PackedRnn pack_lstm(const float *w_ih, const float *w_hh, const float *b_ih, const float *b_hh, int In, int H) {
    PackedRnn P;
    P.K0 = In; P.K0p = round_up(In, 4); P.Kp = round_up(P.K0p + H, PACK_KPAD);
    P.W.assign((size_t) 4 * H * P.Kp, 0.f);
    P.bias.assign((size_t) 4 * H, 0.f);
    for (int j = 0; j < H; j++)
        for (int g = 0; g < 4; g++) {
            float *row = &P.W[(size_t) (4 * j + g) * P.Kp];
            const int src = g * H + j;
            for (int k = 0; k < In; k++) row[k] = w_ih[(size_t) src * In + k];
            for (int k = 0; k < H; k++) row[P.K0p + k] = w_hh[(size_t) src * H + k];
            P.bias[4 * j + g] = b_ih[src] + b_hh[src];
        }
    return P;
}
// PyTorch GRU params (gate order r,z,n) -> rows 4j+{r, z, n_x, n_h}
static PackedRnn pack_gru(const float *w_ih, const float *w_hh, const float *b_ih, const float *b_hh, int In, int H) {
    PackedRnn P;
    P.K0 = In; P.K0p = round_up(In, 4); P.Kp = round_up(P.K0p + H, PACK_KPAD);
    P.W.assign((size_t) 4 * H * P.Kp, 0.f);
    P.bias.assign((size_t) 4 * H, 0.f);
    for (int j = 0; j < H; j++) {
        for (int g = 0; g < 2; g++) {
            float *row = &P.W[(size_t) (4 * j + g) * P.Kp];
            const int src = g * H + j;
            for (int k = 0; k < In; k++) row[k] = w_ih[(size_t) src * In + k];
            for (int k = 0; k < H; k++) row[P.K0p + k] = w_hh[(size_t) src * H + k];
            P.bias[4 * j + g] = b_ih[src] + b_hh[src];
        }
        const int src = 2 * H + j;
        float *rx = &P.W[(size_t) (4 * j + 2) * P.Kp], *rh = &P.W[(size_t) (4 * j + 3) * P.Kp];
        for (int k = 0; k < In; k++) rx[k] = w_ih[(size_t) src * In + k];
        for (int k = 0; k < H; k++) rh[P.K0p + k] = w_hh[(size_t) src * H + k];
        P.bias[4 * j + 2] = b_ih[src];
        P.bias[4 * j + 3] = b_hh[src];
    }
    return P;
}

}  // namespace pb

using namespace pb;

// =====================================================================================================
// Variant network
// =====================================================================================================
static const char *VARIANT_PARAMS[PB_VARIANT_NET_N_PARAMS] = {
    "encoder.weight_ih_l0", "encoder.weight_hh_l0", "encoder.bias_ih_l0", "encoder.bias_hh_l0",
    "encoder.weight_ih_l0_reverse", "encoder.weight_hh_l0_reverse", "encoder.bias_ih_l0_reverse", "encoder.bias_hh_l0_reverse",
    "decoder.weight_ih_l0", "decoder.weight_hh_l0", "decoder.bias_ih_l0", "decoder.bias_hh_l0",
    "decoder.weight_ih_l0_reverse", "decoder.weight_hh_l0_reverse", "decoder.bias_ih_l0_reverse", "decoder.bias_hh_l0_reverse",
    "linear_1.weight", "linear_1.bias", "linear_2.weight", "linear_2.bias", "linear_3.weight", "linear_3.bias",
    "linear_4.weight", "linear_4.bias", "linear_5.weight", "linear_5.bias", "output_layer_type.weight", "output_layer_type.bias"};
static const int64_t VARIANT_NUMEL[PB_VARIANT_NET_N_PARAMS] = {
    1024 * 26, 1024 * 256, 1024, 1024, 1024 * 26, 1024 * 256, 1024, 1024,
    1024 * 512, 1024 * 256, 1024, 1024, 1024 * 512, 1024 * 256, 1024, 1024,
    512 * 16896, 512, 512 * 512, 512, 512 * 512, 512, 512 * 512, 512, 512 * 512, 512, 3 * 512, 3};

extern "C" const char *pb_variant_net_param_name(int i) { return (i >= 0 && i < PB_VARIANT_NET_N_PARAMS) ? VARIANT_PARAMS[i] : nullptr; }
extern "C" int64_t pb_variant_net_param_numel(int i) { return (i >= 0 && i < PB_VARIANT_NET_N_PARAMS) ? VARIANT_NUMEL[i] : -1; }


constexpr int VT = 33, VH = 256;
constexpr int64_t VARIANT_CHUNK = 8448;     // 66 row tiles x 2 directions = 132 k_lstm_layer CTAs = one per H100 SM

extern "C" int pb_variant_net_create(pb_variant_net_t **out, int device, const float *const *P) {
    if (!out || !P) { set_error("null argument"); return PB_ERR_ARG; }
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= device) {
        set_error("no CUDA device %d (found %d): libpepper_b200 has no CPU fallback", device, n);
        return PB_ERR_CUDA;
    }
    for (int i = 0; i < PB_VARIANT_NET_N_PARAMS; i++) if (!P[i]) { set_error("missing parameter %s", VARIANT_PARAMS[i]); return PB_ERR_ARG; }
    PB_CUDA(cudaSetDevice(device));
    auto *N = new pb_variant_net();
    N->device = device;
    TcVariant &T = N->tc;
    for (int d = 0; d < 2; d++) {
        const PackedRnn pe = pack_lstm(P[4 * d + 0], P[4 * d + 1], P[4 * d + 2], P[4 * d + 3], 26, VH);
        const PackedRnn pd = pack_lstm(P[8 + 4 * d + 0], P[8 + 4 * d + 1], P[8 + 4 * d + 2], P[8 + 4 * d + 3], 512, VH);
        PB_TRY(tc_upload_rnn(T.enc[d], pe.W.data(), pe.bias.data(), pe.K0, pe.K0p, VH, pe.Kp, true));
        PB_TRY(tc_upload_rnn(T.dec[d], pd.W.data(), pd.bias.data(), pd.K0, pd.K0p, VH, pd.Kp));
        PB_TRY(tc_upload_rnn_q8(T.decq[d], pd.W.data(), pd.K0, pd.K0p, VH, pd.Kp));
    }
    // linear_1 twice: fp16 hi / lo tiles for mode 1, int8 slices for mode 2
    PB_TRY(tc_upload_lin(T.lin[0], P[16], P[17], 512, VT * 512));
    PB_TRY(tc_upload_q8(T.lin1q, P[16], 512, VT * 512, true));
    for (int i = 1; i < 5; i++) PB_TRY(tc_upload_lin(T.lin[i], P[16 + 2 * i], P[17 + 2 * i], 512, 512));
    PB_TRY(upload(N->out_w, P[26], sizeof(float) * 3 * 512, 0));
    PB_TRY(upload(N->out_b, P[27], sizeof(float) * 3, 0));
    // the int8 guard: weights whose slices would cost a gate or a linear_1 output more than its threshold run the network on
    // the fp16 split instead, with all three products: the two-product recurrent GEMMs of mask 0x1a miss the parity gate on
    // such weights too (an outlier of 100 std in W_hh multiplies the dropped a_lo, DESIGN.md "Int8-slice decoder")
    N->q8_gate_err = std::max(T.decq[0].err, T.decq[1].err);
    N->q8_head_err = T.lin1q.err;
    N->mode = N->q8_gate_err < PB_VARIANT_Q8_MAX_GATE_ERR && N->q8_head_err < PB_VARIANT_Q8_HEAD_MAX_ERR ? 2 : 1;
    if (N->mode == 1) T.lo_mask = 0x1f;
    *out = N;
    return PB_OK;
}

extern "C" int pb_variant_net_q8_guard(pb_variant_net_t *N, double *gate_err, int *mode) {
    if (!N) { set_error("null network"); return PB_ERR_ARG; }
    if (gate_err) *gate_err = N->q8_gate_err;
    if (mode) *mode = N->mode;
    return PB_OK;
}

extern "C" int pb_variant_net_q8_head_err(pb_variant_net_t *N, double *head_err) {
    if (!N || !head_err) { set_error("null argument"); return PB_ERR_ARG; }
    *head_err = N->q8_head_err;
    return PB_OK;
}

extern "C" int pb_variant_net_destroy(pb_variant_net_t *N) {
    if (!N) return PB_OK;
    TcVariant &T = N->tc;
    for (int d = 0; d < 2; d++) {
        TcRnn *rnn[] = {&T.enc[d], &T.dec[d]};
        for (auto *r : rnn) { r->w_hi.release(); r->w_lo.release(); r->wh_hi.release(); r->wh_lo.release(); r->bias.release(); }
        T.decq[d].w1.release(); T.decq[d].w0.release(); T.decq[d].col_scale.release();
    }
    T.lin1q.w1.release(); T.lin1q.w0.release(); T.lin1q.col_scale.release();
    for (auto &l : T.lin) { l.w_hi.release(); l.w_lo.release(); l.bias.release(); }
    DevBuf *bufs[] = {&N->out_w, &N->out_b, &N->img, &N->probs, &T.img_op, &T.yenc_hi, &T.yenc_lo, &T.ydec_hi, &T.ydec_lo, &T.ydec_q,
                      &T.c, &T.act_hi[0], &T.act_hi[1], &T.act_lo[0], &T.act_lo[1], &T.final_f32};
    for (auto *b : bufs) b->release();
    delete N;
    return PB_OK;
}

extern "C" int pb_variant_net_set_mode(pb_variant_net_t *N, int mode) {
    if (!N) return PB_ERR_ARG;
    if (mode != 1 && mode != 2) {
        set_error("mode %d unknown (1 = tensor-core hi/lo x3, 2 = tensor cores with the decoder LSTM and linear_1 on int8 slices)", mode);
        return PB_ERR_ARG;
    }
    N->mode = mode;
    return PB_OK;
}
// experiments (DESIGN.md "two-product variant"): which GEMMs keep the third tensor-core product.  The mask selects among the
// fp16 split's products, so a network in mode 2 goes back to mode 1, where every bit applies.
extern "C" int pb_variant_net_set_lo_mask(pb_variant_net_t *N, int mask) {
    if (!N) { set_error("null network"); return PB_ERR_ARG; }
    N->tc.lo_mask = mask & 0x1f;
    if (N->mode == 2) N->mode = 1;
    return PB_OK;
}
extern "C" int pb_polish_net_set_lo_mask(pb_polish_net_t *N, int mask) {
    if (!N) { set_error("null network"); return PB_ERR_ARG; }
    N->tc.lo_mask = mask & 0x7;
    return PB_OK;
}
extern "C" int pb_variant_net_launches(pb_variant_net_t *N, int64_t *n) {
    if (!N || !n) return PB_ERR_ARG;
    *n = N->launches;
    return PB_OK;
}

static int variant_forward(pb_variant_net_t *N, const int8_t *d_images, int64_t n, float *d_probs, float *d_hidden_dbg,
                           const pb::OutSink &sink, void *stream_);

extern "C" int pb_variant_net_forward_device(pb_variant_net_t *N, const int8_t *d_images, int64_t n, float *d_probs,
                                             float *d_hidden_dbg, void *stream_) {
    return variant_forward(N, d_images, n, d_probs, d_hidden_dbg, pb::OutSink{}, stream_);
}

extern "C" int pb_variant_net_forward_records_device(pb_variant_net_t *N, const int8_t *d_images, int64_t n, float *d_probs,
                                                     const pb_candidate_columns_t *cols, pb_pred_record_t *d_records, void *stream_) {
    pb::OutSink S{};
    if (d_records) {
        if (!cols || !cols->positions || !cols->region_of || !cols->depths || !cols->freqs || !cols->keys) {
            set_error("record sink needs all candidate columns"); return PB_ERR_ARG;
        }
        S.cols = *cols; S.records = d_records;
    }
    return variant_forward(N, d_images, n, d_probs, nullptr, S, stream_);
}

static int variant_forward(pb_variant_net_t *N, const int8_t *d_images, int64_t n, float *d_probs, float *d_hidden_dbg,
                           const pb::OutSink &sink, void *stream_) {
    if (!N || (n > 0 && (!d_images || !d_probs))) { set_error("null argument"); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    PB_CUDA(cudaSetDevice(N->device));
    N->launches = 0;
    for (int64_t b0 = 0; b0 < n; b0 += VARIANT_CHUNK) {
        const int64_t B = std::min(VARIANT_CHUNK, n - b0);
        PB_TRY(variant_forward_tc(N, d_images + b0 * VT * 26, B, d_probs + b0 * 3, d_hidden_dbg ? d_hidden_dbg + b0 * VT * 512 : nullptr,
                                  st, sink.at(b0)));
    }
    return PB_OK;
}

extern "C" int pb_variant_net_forward_host(pb_variant_net_t *N, const int8_t *h_images, int64_t n, float *h_probs,
                                           float *h_hidden_dbg, void *stream_) {
    if (!N) return PB_ERR_ARG;
    cudaStream_t st = (cudaStream_t) stream_;
    PB_CUDA(cudaSetDevice(N->device));
    if (n <= 0) return PB_OK;
    DevBuf hid;
    PB_TRY(N->img.reserve((size_t) n * VT * 26));
    PB_TRY(N->probs.reserve(sizeof(float) * n * 3));
    if (h_hidden_dbg) PB_TRY(hid.reserve(sizeof(float) * n * VT * 512));
    PB_CUDA(cudaMemcpyAsync(N->img.p, h_images, (size_t) n * VT * 26, cudaMemcpyHostToDevice, st));
    int rc = pb_variant_net_forward_device(N, N->img.as<int8_t>(), n, N->probs.as<float>(), h_hidden_dbg ? hid.as<float>() : nullptr, stream_);
    if (rc == PB_OK) {
        cudaError_t e = cudaMemcpyAsync(h_probs, N->probs.p, sizeof(float) * n * 3, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess && h_hidden_dbg) e = cudaMemcpyAsync(h_hidden_dbg, hid.p, sizeof(float) * n * VT * 512, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("variant net copy back: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    }
    hid.release();
    return rc;
}

// =====================================================================================================
// Polish network
// =====================================================================================================
static const char *POLISH_PARAMS[PB_POLISH_NET_N_PARAMS] = {
    "gru_encoder.weight_ih_l0", "gru_encoder.weight_hh_l0", "gru_encoder.bias_ih_l0", "gru_encoder.bias_hh_l0",
    "gru_encoder.weight_ih_l0_reverse", "gru_encoder.weight_hh_l0_reverse", "gru_encoder.bias_ih_l0_reverse", "gru_encoder.bias_hh_l0_reverse",
    "gru_decoder.weight_ih_l0", "gru_decoder.weight_hh_l0", "gru_decoder.bias_ih_l0", "gru_decoder.bias_hh_l0",
    "gru_decoder.weight_ih_l0_reverse", "gru_decoder.weight_hh_l0_reverse", "gru_decoder.bias_ih_l0_reverse", "gru_decoder.bias_hh_l0_reverse",
    "dense1.weight", "dense1.bias"};
static const int64_t POLISH_NUMEL[PB_POLISH_NET_N_PARAMS] = {
    384 * 10, 384 * 128, 384, 384, 384 * 10, 384 * 128, 384, 384,
    384 * 256, 384 * 128, 384, 384, 384 * 256, 384 * 128, 384, 384, 5 * 256, 5};
extern "C" const char *pb_polish_net_param_name(int i) { return (i >= 0 && i < PB_POLISH_NET_N_PARAMS) ? POLISH_PARAMS[i] : nullptr; }
extern "C" int64_t pb_polish_net_param_numel(int i) { return (i >= 0 && i < PB_POLISH_NET_N_PARAMS) ? POLISH_NUMEL[i] : -1; }

constexpr int PH = 128, PSEQ = 1000, PNWIN = 19;

extern "C" int pb_polish_net_create(pb_polish_net_t **out, int device, const float *const *P) {
    if (!out || !P) { set_error("null argument"); return PB_ERR_ARG; }
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= device) {
        set_error("no CUDA device %d (found %d): libpepper_b200 has no CPU fallback", device, n);
        return PB_ERR_CUDA;
    }
    for (int i = 0; i < PB_POLISH_NET_N_PARAMS; i++) if (!P[i]) { set_error("missing parameter %s", POLISH_PARAMS[i]); return PB_ERR_ARG; }
    PB_CUDA(cudaSetDevice(device));
    auto *N = new pb_polish_net();
    N->device = device;
    for (int d = 0; d < 2; d++) {
        const PackedRnn pe = pack_gru(P[4 * d + 0], P[4 * d + 1], P[4 * d + 2], P[4 * d + 3], 10, PH);
        const PackedRnn pd = pack_gru(P[8 + 4 * d + 0], P[8 + 4 * d + 1], P[8 + 4 * d + 2], P[8 + 4 * d + 3], 256, PH);
        PB_TRY(tc_upload_rnn(N->tc.enc[d], pe.W.data(), pe.bias.data(), pe.K0, pe.K0p, PH, pe.Kp));
        PB_TRY(tc_upload_rnn(N->tc.dec[d], pd.W.data(), pd.bias.data(), pd.K0, pd.K0p, PH, pd.Kp));
    }
    PB_TRY(N->dW.reserve(sizeof(float) * 5 * 256));
    PB_TRY(N->dB.reserve(sizeof(float) * 8));
    PB_CUDA(cudaMemcpy(N->dW.p, P[16], sizeof(float) * 5 * 256, cudaMemcpyHostToDevice));
    PB_CUDA(cudaMemcpy(N->dB.p, P[17], sizeof(float) * 5, cudaMemcpyHostToDevice));
    *out = N;
    return PB_OK;
}

extern "C" int pb_polish_net_destroy(pb_polish_net_t *N) {
    if (!N) return PB_OK;
    TcPolish &T = N->tc;
    for (int d = 0; d < 2; d++) {
        TcRnn *rnn[] = {&T.enc[d], &T.dec[d]};
        for (auto *r : rnn) { r->w_hi.release(); r->w_lo.release(); r->bias.release(); }
    }
    DevBuf *bufs[] = {&N->dW, &N->dB, &N->acc, &N->img, &N->bases, &N->phred, &T.img_op, &T.yenc_hi, &T.yenc_lo, &T.ydec_hi, &T.ydec_lo,
                      &T.zero, &T.flags};
    for (auto *b : bufs) b->release();
    delete N;
    return PB_OK;
}
extern "C" int pb_polish_net_launches(pb_polish_net_t *N, int64_t *n) {
    if (!N || !n) return PB_ERR_ARG;
    *n = N->launches;
    return PB_OK;
}

extern "C" int pb_polish_net_forward_device(pb_polish_net_t *N, const uint8_t *d_images, int64_t n, uint8_t *d_bases,
                                            uint8_t *d_phred, float *d_hidden_dbg, float *d_acc_dbg, void *stream_) {
    if (!N || (n > 0 && (!d_images || !d_bases || !d_phred))) { set_error("null argument"); return PB_ERR_ARG; }
    cudaStream_t st = (cudaStream_t) stream_;
    PB_CUDA(cudaSetDevice(N->device));
    N->launches = 0;
    int sms = 0;
    PB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, N->device));
    // a window layer is one k_gru_layer launch of one CTA per (direction, row tile), so sms / 2 row tiles fill the GPU
    const int64_t chunk = std::max<int64_t>(1, sms / 2) * 128;
    for (int64_t b0 = 0; b0 < n; b0 += chunk) {
        const int64_t B = std::min(chunk, n - b0);
        PB_TRY(N->acc.reserve(sizeof(float) * B * PSEQ * 5));
        PB_CUDA(cudaMemsetAsync(N->acc.p, 0, sizeof(float) * B * PSEQ * 5, st));
        PB_TRY(polish_forward_tc(N, d_images + b0 * PSEQ * 10, B, n, b0, d_hidden_dbg, st));
        k_polish_finalize<<<(unsigned) ceil_div(B * PSEQ, 256), 256, 0, st>>>(N->acc.as<float>(), d_bases + b0 * PSEQ, d_phred + b0 * PSEQ, B);
        N->launches++;
        if (d_acc_dbg)
            PB_CUDA(cudaMemcpyAsync(d_acc_dbg + b0 * PSEQ * 5, N->acc.p, sizeof(float) * B * PSEQ * 5, cudaMemcpyDeviceToDevice, st));
        PB_CUDA(cudaGetLastError());
    }
    return PB_OK;
}

extern "C" int pb_polish_net_forward_host(pb_polish_net_t *N, const uint8_t *h_images, int64_t n, uint8_t *h_bases,
                                          uint8_t *h_phred, float *h_hidden_dbg, float *h_acc_dbg, void *stream_) {
    if (!N) return PB_ERR_ARG;
    cudaStream_t st = (cudaStream_t) stream_;
    PB_CUDA(cudaSetDevice(N->device));
    if (n <= 0) return PB_OK;
    DevBuf hid, accd;
    PB_TRY(N->img.reserve((size_t) n * PSEQ * 10));
    PB_TRY(N->bases.reserve((size_t) n * PSEQ));
    PB_TRY(N->phred.reserve((size_t) n * PSEQ));
    if (h_hidden_dbg) PB_TRY(hid.reserve(sizeof(float) * PNWIN * n * 2 * PH));
    if (h_acc_dbg) PB_TRY(accd.reserve(sizeof(float) * n * PSEQ * 5));
    PB_CUDA(cudaMemcpyAsync(N->img.p, h_images, (size_t) n * PSEQ * 10, cudaMemcpyHostToDevice, st));
    int rc = pb_polish_net_forward_device(N, N->img.as<uint8_t>(), n, N->bases.as<uint8_t>(), N->phred.as<uint8_t>(),
                                          h_hidden_dbg ? hid.as<float>() : nullptr, h_acc_dbg ? accd.as<float>() : nullptr, stream_);
    if (rc == PB_OK) {
        cudaError_t e = cudaMemcpyAsync(h_bases, N->bases.p, (size_t) n * PSEQ, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(h_phred, N->phred.p, (size_t) n * PSEQ, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess && h_hidden_dbg) e = cudaMemcpyAsync(h_hidden_dbg, hid.p, sizeof(float) * PNWIN * n * 2 * PH, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess && h_acc_dbg) e = cudaMemcpyAsync(h_acc_dbg, accd.p, sizeof(float) * n * PSEQ * 5, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("polish net copy back: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    }
    hid.release(); accd.release();
    return rc;
}
