// Host side of the tensor-core (wgmma) network paths (modes 1 and 2): weight / operand tiling, per-layer launch sequences, and a
// GEMM self-test entry point.  Device code: tc_gemm.cuh.
#include "handles.cuh"
#include "tc_gemm.cuh"
#include <vector>
#include <algorithm>
#include <cmath>

using namespace pb;
using tc::Args;
using tc::Dir;
using tc::Seg;
using tc::TILE_ELEMS;
typedef pb::tc::op_t bf16;      // 16-bit operand element (fp16 by default, bf16 with -DPB_OPERAND_BF16)

namespace pb {

static inline uint16_t f2bf(float f) { return tc::op_bits(f); }      // round to nearest even into the operand type
static inline float bf2f(uint16_t h) { return tc::op_val(h); }

// element (r, k) of a matrix tiled in TR-row x 32-k tiles [rt][kt][4][TR][8], KT k-tiles per row tile
static inline int64_t tiled_index(int64_t r, int64_t k, int64_t KT, int64_t TR) {
    return ((r / TR) * KT + k / 32) * (TR * 32) + ((k % 32) / 8) * (TR * 8) + (r % TR) * 8 + (k % 8);
}

// row-major [rows][K] fp32 (rows % 128 == 0 after padding, K % 32 == 0 after padding) -> hi / lo tiles [rt][kt][4][128][8]
static void tile_matrix(const float *src, int64_t rows, int64_t K, int64_t rows_p, int64_t Kp, std::vector<uint16_t> &hi, std::vector<uint16_t> &lo,
                        int64_t TR = 128 /* rows per tile: 128 for A operands, 256 for the weights of the persistent kernel */) {
    const int64_t RT = rows_p / TR, KT = Kp / 32;
    hi.assign((size_t) (RT * KT * TR * 32), 0);
    lo.assign((size_t) (RT * KT * TR * 32), 0);
    for (int64_t r = 0; r < rows; r++)
        for (int64_t k = 0; k < K; k++) {
            const float v = src[r * K + k];
            const uint16_t h = f2bf(v);
            const uint16_t l = f2bf(v - bf2f(h));
            const int64_t o = tiled_index(r, k, KT, TR);
            hi[(size_t) o] = h;
            lo[(size_t) o] = l;
        }
}

static int upload_tiles(DevBuf &dhi, DevBuf &dlo, const std::vector<uint16_t> &hi, const std::vector<uint16_t> &lo) {
    PB_TRY(dhi.reserve(hi.size() * 2));
    PB_TRY(dlo.reserve(lo.size() * 2));
    PB_CUDA(cudaMemcpy(dhi.p, hi.data(), hi.size() * 2, cudaMemcpyHostToDevice));
    PB_CUDA(cudaMemcpy(dlo.p, lo.data(), lo.size() * 2, cudaMemcpyHostToDevice));
    return PB_OK;
}

// The power of two s with max |s W| in (2^14, 2^15] (fp16 holds up to 65,504).  An fp16 w_lo is subnormal below 2^-14, i.e.
// for |s w| < 2^-3, where it carries an absolute error of up to 2^-25: scaled, that error is 2^-25 / s of the unscaled weight,
// and the split keeps its 22 bits for every weight down to 2^-17 of the matrix maximum.  A heavy-tailed matrix (one weight
// at 100x the std of the rest) needs that range: at max |s W| ~ 1, most of its weights' w_lo would be subnormal.
static float pow2_scale(const float *w, size_t n) {
    float m = 0.f;
    for (size_t i = 0; i < n; i++) m = std::max(m, std::fabs(w[i]));
    if (!(m > 0.f) || !std::isfinite(m)) return 1.f;
    int e;
    const float f = std::frexp(m, &e);                      // m = f 2^e, f in [1/2, 1)
    e = std::min(std::max(f == 0.5f ? e - 1 : e, -60), 60); // ceil(log2 m)
    return std::ldexp(1.f, 15 - e);
}

// weights of one RNN direction, packed rows 4j+g (nets.cu pack_lstm / pack_gru) with K = [x | pad32 | h]; x-part and h-part
// share one scale.  half_tiles: also in 128-row tiles (wh_hi / wh_lo), whose k-tiles are the single 8 KB pieces that
// k_lstm_layer_enc's ring stages take (a 128-row half of a 256-row tile is 4 pieces of 2 KB, one per 8-k chunk)
int tc_upload_rnn(TcRnn &T, const float *Wp /* [4H][Kp_src] */, const float *bias /* [4H] */, int K0, int K0p_src, int H, int Kp_src,
                  bool half_tiles) {
    const int K0p = (K0 + 31) / 32 * 32;
    const int Kp = K0p + H;
    std::vector<float> W((size_t) 4 * H * Kp, 0.f);
    for (int n = 0; n < 4 * H; n++) {
        for (int k = 0; k < K0; k++) W[(size_t) n * Kp + k] = Wp[(size_t) n * Kp_src + k];
        for (int k = 0; k < H; k++) W[(size_t) n * Kp + K0p + k] = Wp[(size_t) n * Kp_src + K0p_src + k];
    }
    T.scale = pow2_scale(W.data(), W.size());
    for (float &v : W) v *= T.scale;
    std::vector<uint16_t> hi, lo;
    tile_matrix(W.data(), 4 * H, Kp, 4 * H, Kp, hi, lo, 256);
    T.nkt_x = K0p / 32; T.nkt_h = H / 32;
    PB_TRY(upload(T.bias, bias, sizeof(float) * 4 * H, 0));
    PB_TRY(upload_tiles(T.w_hi, T.w_lo, hi, lo));
    if (!half_tiles) return PB_OK;
    tile_matrix(W.data(), 4 * H, Kp, 4 * H, Kp, hi, lo, 128);
    return upload_tiles(T.wh_hi, T.wh_lo, hi, lo);
}
int tc_upload_lin(TcLin &T, const float *w, const float *bias, int N, int K) {
    T.scale = pow2_scale(w, (size_t) N * K);
    std::vector<float> W(w, w + (size_t) N * K);
    for (float &v : W) v *= T.scale;
    std::vector<uint16_t> hi, lo;
    const int Np = (N + 255) / 256 * 256, Kp = (K + 31) / 32 * 32;
    tile_matrix(W.data(), N, K, Np, Kp, hi, lo, 256);
    T.nkt = Kp / 32;
    PB_TRY(upload(T.bias, bias, sizeof(float) * N, 0));
    return upload_tiles(T.w_hi, T.w_lo, hi, lo);
}

// 16-bit fixed point q = rint(v * s) as two int8 slices q = 256 q1 + q0 (tc_gemm.cuh, "int8-slice operands")
static inline void qsplit(double v_times_s, int8_t &q1, int8_t &q0) {
    const int q = (int) std::nearbyint(v_times_s);
    const int hi = (q + 128) >> 8;
    q1 = (int8_t) hi;
    q0 = (int8_t) (q - 256 * hi);
}
// byte offset of element (r, k) in a [rt][kt][4][128][16] slice image with KT k-tiles of 64 per row tile
static inline int64_t qtiled_index(int64_t r, int64_t k, int64_t KT) {
    return ((r / 128) * KT + k / 64) * tc::QTILE_BYTES + ((k % 64) / 16) * 2048 + (r % 128) * 16 + (k % 16);
}

// W [N][K] row-major -> the slice images of TcQ8 (tiled with qtiled_index, K / 64 k-tiles per 128-row n-tile) and the column
// scales.  row_err[n]: the weight-only estimate of the error the slices add to output n's pre-activation (DESIGN.md
// "Int8-slice decoder" and "linear_1 on int8 slices"),
//   e_n = sqrt(sum_k (w_k / sw_n - W_k)^2 + (128^2 / 3) / 32512^2 sum_k (w0_k / sw_n)^2 [+ sum_k W_k^2 / (12 32512^2)])
// (weight rounding at |a_k| = 1, plus the dropped a0 w0 product with a0 uniform over its 8 bits; a_quant adds the rounding of
// fp32 activations to 1 / 32512 steps, which linear_1's fp16 path does not have).
static void pack_q8(const float *W, int N, int K, bool a_quant, std::vector<int8_t> &w1, std::vector<int8_t> &w0,
                    std::vector<float> &cs, std::vector<double> &row_err) {
    const int KT = K / tc::QK;
    const double qs2 = (double) tc::QSCALE * tc::QSCALE;
    const double a0_var = 128.0 * 128.0 / 3.0 / qs2;
    w1.assign((size_t) N * K, 0); w0.assign((size_t) N * K, 0);
    cs.assign(N, 0.f); row_err.assign(N, 0.0);
    for (int n = 0; n < N; n++) {
        const float *x = W + (size_t) n * K;
        double m = 0.0;
        for (int k = 0; k < K; k++) m = std::max(m, (double) std::fabs(x[k]));
        const double sw = m > 0.0 && std::isfinite(m) ? tc::QSCALE / m : 1.0;
        cs[n] = (float) (256.0 / (tc::QSCALE * sw));
        double e_round = 0.0, e_drop = 0.0, sq = 0.0;
        for (int k = 0; k < K; k++) {
            const int64_t o = qtiled_index(n, k, KT);
            const double w = x[k];
            int8_t &s1 = w1[(size_t) o], &s0 = w0[(size_t) o];
            qsplit(w * sw, s1, s0);
            const double r = (256.0 * s1 + s0) / sw - w, d = s0 / sw;
            e_round += r * r;
            e_drop += d * d;
            sq += w * w;
        }
        row_err[n] = std::sqrt(e_round + a0_var * e_drop + (a_quant ? sq / (12.0 * qs2) : 0.0));
    }
}

int tc_upload_q8(TcQ8 &T, const float *W, int N, int K, bool a_quant) {
    if (K % tc::QK || N % tc::QN) { set_error("int8 slice packing needs N %% 128 == 0 and K %% 64 == 0"); return PB_ERR_ARG; }
    std::vector<int8_t> w1, w0;
    std::vector<float> cs;
    std::vector<double> err;
    pack_q8(W, N, K, a_quant, w1, w0, cs, err);
    T.err = *std::max_element(err.begin(), err.end());
    PB_TRY(T.w1.reserve(w1.size()));
    PB_TRY(T.w0.reserve(w0.size()));
    PB_TRY(T.col_scale.reserve(sizeof(float) * N));
    PB_CUDA(cudaMemcpy(T.w1.p, w1.data(), w1.size(), cudaMemcpyHostToDevice));
    PB_CUDA(cudaMemcpy(T.w0.p, w0.data(), w0.size(), cudaMemcpyHostToDevice));
    PB_CUDA(cudaMemcpy(T.col_scale.p, cs.data(), sizeof(float) * N, cudaMemcpyHostToDevice));
    return PB_OK;
}
// the decoder direction's weights for k_lstm_layer_q8: rows 4j+g of Wp [4H][Kp_src] with K = [x | pad32 | h] -> K = [x | h]
int tc_upload_rnn_q8(TcQ8 &T, const float *Wp, int K0, int K0p_src, int H, int Kp_src) {
    const int K = K0 + H, N = 4 * H;
    std::vector<float> W((size_t) N * K);
    for (int n = 0; n < N; n++) {
        std::copy(Wp + (size_t) n * Kp_src, Wp + (size_t) n * Kp_src + K0, W.begin() + (size_t) n * K);
        std::copy(Wp + (size_t) n * Kp_src + K0p_src, Wp + (size_t) n * Kp_src + K0p_src + H, W.begin() + (size_t) n * K + K0);
    }
    return tc_upload_q8(T, W.data(), N, K, false);
}

static int g_num_sms = 0;

// persistent 128x256-tile kernel (weights packed in 256-row tiles); `nt128` = number of 128-column tiles = N / 128.
// One CTA per SM, or at most `max_ctas` (> 0), so that every CTA walks several tiles.
template <int EPI>
static int launch_tc(const Args &A, int mt, int nt128, int ndir, cudaStream_t st, int max_ctas = 0) {
    static bool attr_set = false;
    if (!attr_set) {
        PB_CUDA(cudaFuncSetAttribute(tc::k_tc_gemm_p<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::PSMEM_BYTES));
        attr_set = true;
    }
    if (g_num_sms == 0) {
        int dev = 0;
        PB_CUDA(cudaGetDevice(&dev));
        PB_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
    }
    if (nt128 % 2) { set_error("tensor-core path needs N %% 256 == 0"); return PB_ERR_ARG; }
    const int nt = nt128 / 2;
    const int tiles = mt * nt * ndir;
    const int ctas = std::min(tiles, max_ctas > 0 ? std::min(max_ctas, g_num_sms) : g_num_sms);
    tc::k_tc_gemm_p<EPI><<<(unsigned) ctas, tc::PG_THREADS, tc::PSMEM_BYTES, st>>>(A, mt, nt, ndir);
    return PB_OK;
}
static Dir empty_dir() {
    Dir D;
    memset(&D, 0, sizeof(D));
    return D;
}

// ------------------------------------------------------------------------------------------------- variant
constexpr int VT = 33, VH = 256;
// bytes per row tile of one slice of a 512-feature sequence (tc_gemm.cuh QSeq): 33 steps x 8 k-tiles.  Both slices of a
// sequence take as many bytes as its fp16 lo tiles, so the encoder's go into T.yenc_lo (q1, then q0 at Mt * q_mt_bytes()).
static constexpr int64_t q_mt_bytes() { return (int64_t) VT * 8 * tc::QTILE_BYTES; }

#ifdef PB_LSTM_TRACE
// Timing build only: the stamps of the latest launch of each variant LSTM layer (layer 0 words, then layer 1), on the
// device that ran it.  pb_lstm_trace_copy is exported by these builds alone (scripts/trace_lstm_layer.py).
static uint64_t *g_lstm_trace = nullptr;
static int lstm_trace_buffer(int layer, uint64_t **out) {
    if (!g_lstm_trace) PB_CUDA(cudaMalloc(&g_lstm_trace, sizeof(uint64_t) * 2 * tc::lstm_trace_words(VT)));
    *out = g_lstm_trace + layer * tc::lstm_trace_words(VT);
    return PB_OK;
}
extern "C" int pb_lstm_trace_copy(uint64_t *host, int64_t n_words) {
    if (!g_lstm_trace) { set_error("no k_lstm_layer launch has been traced"); return PB_ERR_STATE; }
    if (n_words != 2 * tc::lstm_trace_words(VT)) { set_error("trace holds 2 x %lld words", (long long) tc::lstm_trace_words(VT)); return PB_ERR_ARG; }
    PB_CUDA(cudaDeviceSynchronize());
    PB_CUDA(cudaMemcpy(host, g_lstm_trace, sizeof(uint64_t) * n_words, cudaMemcpyDeviceToHost));
    return PB_OK;
}
#endif

// One bidirectional LSTM layer of the variant network over its 33 steps, reading T.img_op (layer 0) or T.yenc (layer 1)
// and writing T.yenc / T.ydec (+ the optional fp32 copy y_f32 [B][33][512]); the cell state ends in T.c.  lo_x / lo_h:
// the a_lo x w_hi product of the x-part / h-part runs (the int8 images of layer 0 have no lo operand).  persist: one
// launch (the forward pass), or 33 launches of the per-step k_tc_gemm_p<EPI_LSTM> path, the reference that
// pb_test_variant_lstm_layer offers for it.  The persistent encoder layer with a hi-only h-part runs k_lstm_layer_enc (h kept
// in shared memory); k_lstm_layer runs the rest (the decoder of mode 1, and an encoder h-part with all three products,
// whose hi + lo h would need 128 KB per step buffer).  q8 (layer 0, persistent, hi-only h-part): the layer writes the int8
// slices of h for k_lstm_layer_q8 into T.yenc_lo instead of the fp16 lo tiles.
static int variant_lstm_layer_tc(pb_variant_net *N, int layer, int64_t B, bool lo_x, bool lo_h, bool persist, float *y_f32,
                                 cudaStream_t st, bool q8 = false) {
    TcVariant &T = N->tc;
    const int64_t Mt = ceil_div(B, 128), Bp = Mt * 128;
    PB_CUDA(cudaMemsetAsync(T.c.p, 0, sizeof(float) * 2 * VH * Bp, st));
    bf16 *y_hi = layer == 0 ? T.yenc_hi.as<bf16>() : T.ydec_hi.as<bf16>();
    bf16 *y_lo = layer == 0 ? T.yenc_lo.as<bf16>() : T.ydec_lo.as<bf16>();
    const bf16 *x_hi = layer == 0 ? T.img_op.as<bf16>() : T.yenc_hi.as<bf16>();
    const bf16 *x_lo = layer == 0 ? nullptr : T.yenc_lo.as<bf16>();
    const int x_nkt = layer == 0 ? 1 : 16;
    const int64_t x_mt_stride = (int64_t) VT * x_nkt * TILE_ELEMS, y_mt_stride = (int64_t) VT * 16 * TILE_ELEMS;
    TcRnn *W = layer == 0 ? T.enc : T.dec;
    for (int d = 0; d < 2; d++)
        if (W[d].nkt_x != x_nkt || W[d].nkt_h != 8) { set_error("unexpected packed LSTM weight shape"); return PB_ERR_STATE; }
    if (persist) {
        // one launch per layer: every CTA keeps its (direction, row tile) for all 33 steps
        const bool enc = layer == 0 && !lo_h;
        tc::LstmLayer L;
        memset(&L, 0, sizeof(L));
        L.x_hi = x_hi; L.x_lo = x_lo; L.x_mt_stride = x_mt_stride; L.x_nkt = x_nkt;
        for (int d = 0; d < 2; d++) {
            L.w_hi[d] = W[d].w_hi.as<bf16>(); L.w_lo[d] = W[d].w_lo.as<bf16>();
            L.wh_hi[d] = W[d].wh_hi.as<bf16>(); L.wh_lo[d] = W[d].wh_lo.as<bf16>();
            L.bias[d] = W[d].bias.as<float>();
            L.inv_scale[d] = 1.f / W[d].scale;
            L.c[d] = T.c.as<float>() + (int64_t) d * VH * Bp;
        }
        L.y_hi = y_hi; L.y_lo = y_lo; L.y_mt_stride = y_mt_stride;
        if (y_f32) { L.y_f32 = y_f32; L.ldy = (int64_t) VT * 512; }
        L.M = (int) B; L.n_mt = (int) Mt; L.T = VT;
        L.lo_x = lo_x; L.lo_h = lo_h;
        if (enc && !L.wh_hi[0]) { set_error("encoder weights without their half-tile packing"); return PB_ERR_STATE; }
        if (q8) {
            if (!enc) { set_error("int8 slice output: encoder layer with a hi-only h-part"); return PB_ERR_STATE; }
            L.q1 = T.yenc_lo.as<int8_t>(); L.q0 = L.q1 + Mt * q_mt_bytes(); L.q_mt_stride = q_mt_bytes();
        }
#ifdef PB_LSTM_TRACE
        PB_TRY(lstm_trace_buffer(layer, &L.trace));
        PB_CUDA(cudaMemsetAsync(L.trace, 0, sizeof(uint64_t) * tc::lstm_trace_words(VT), st));
#endif
        static bool attr_set = false;
        if (!attr_set) {
            PB_CUDA(cudaFuncSetAttribute(tc::k_lstm_layer, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::LSTM_SMEM_BYTES));
            PB_CUDA(cudaFuncSetAttribute(tc::k_lstm_layer_enc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::ESMEM_BYTES));
            PB_CUDA(cudaFuncSetAttribute(tc::k_lstm_layer_enc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::ESMEM_BYTES));
            attr_set = true;
        }
        if (q8) tc::k_lstm_layer_enc<true><<<(unsigned) (2 * Mt), tc::LSTM_THREADS, tc::ESMEM_BYTES, st>>>(L);
        else if (enc) tc::k_lstm_layer_enc<false><<<(unsigned) (2 * Mt), tc::LSTM_THREADS, tc::ESMEM_BYTES, st>>>(L);
        else tc::k_lstm_layer<<<(unsigned) (2 * Mt), tc::LSTM_THREADS, tc::LSTM_SMEM_BYTES, st>>>(L);
        N->launches++;
        return PB_OK;
    }
    if (q8) { set_error("int8 slice output needs the persistent encoder kernel"); return PB_ERR_STATE; }
    for (int t = 0; t < VT; t++) {
        Args A;
        A.M = (int) B; A.N = 4 * VH;
        for (int d = 0; d < 2; d++) {
            const int tt = d == 0 ? t : VT - 1 - t;
            const int tp = d == 0 ? tt - 1 : tt + 1;
            Dir D = empty_dir();
            D.seg[0].hi = x_hi + (int64_t) tt * x_nkt * TILE_ELEMS; D.seg[0].lo = (x_lo && lo_x) ? x_lo + (int64_t) tt * x_nkt * TILE_ELEMS : nullptr;
            D.seg[0].mt_stride = x_mt_stride; D.seg[0].nkt = x_nkt;
            if (t > 0) {
                D.seg[1].hi = y_hi + ((int64_t) tp * 16 + d * 8) * TILE_ELEMS; D.seg[1].lo = lo_h ? y_lo + ((int64_t) tp * 16 + d * 8) * TILE_ELEMS : nullptr;
                D.seg[1].mt_stride = y_mt_stride; D.seg[1].nkt = 8;
            }
            D.w_hi = W[d].w_hi.as<bf16>(); D.w_lo = W[d].w_lo.as<bf16>(); D.w_nkt = W[d].nkt_x + W[d].nkt_h;
            D.bias = W[d].bias.as<float>();
            D.inv_scale = 1.f / W[d].scale;
            D.c = T.c.as<float>() + (int64_t) d * VH * Bp;
            D.y_hi = y_hi; D.y_lo = y_lo; D.y_mt_stride = y_mt_stride; D.y_kt0 = tt * 16 + d * 8;
            if (y_f32) { D.y_f32 = y_f32 + (int64_t) tt * 512 + d * VH; D.ldy = (int64_t) VT * 512; }
            A.d[d] = D;
        }
        PB_TRY(launch_tc<tc::EPI_LSTM>(A, (int) Mt, 4 * VH / 128, 2, st));
        N->launches++;
    }
    return PB_OK;
}

// The int8-slice decoder layer (mode 2): x = the encoder's slices in T.yenc_lo, h slices in T.ydec_q (its own h-part and
// linear_1's A operand) (+ the optional fp32 copy).  steps: time steps per k_lstm_layer_q8 launch, VT for the forward pass;
// fewer cut the layer into launches that hand h and c over through HBM, the reference for the in-kernel hand-off
// (pb_test_variant_lstm_q8).
static int variant_dec_q8(pb_variant_net *N, int64_t B, int steps, float *y_f32, cudaStream_t st) {
    TcVariant &T = N->tc;
    const int64_t Mt = ceil_div(B, 128), Bp = Mt * 128;
    PB_CUDA(cudaMemsetAsync(T.c.p, 0, sizeof(float) * 2 * VH * Bp, st));
    tc::LstmLayerQ L;
    memset(&L, 0, sizeof(L));
    L.x1 = T.yenc_lo.as<int8_t>(); L.x0 = L.x1 + Mt * q_mt_bytes();
    L.q1 = T.ydec_q.as<int8_t>(); L.q0 = L.q1 + Mt * q_mt_bytes();
    L.q_mt_stride = q_mt_bytes();
    for (int d = 0; d < 2; d++) {
        L.w1[d] = T.decq[d].w1.as<int8_t>(); L.w0[d] = T.decq[d].w0.as<int8_t>();
        L.bias[d] = T.dec[d].bias.as<float>();
        L.col_scale[d] = T.decq[d].col_scale.as<float>();
        L.c[d] = T.c.as<float>() + (int64_t) d * VH * Bp;
    }
    if (y_f32) { L.y_f32 = y_f32; L.ldy = (int64_t) VT * 512; }
    L.M = (int) B; L.n_mt = (int) Mt; L.T = VT;
#ifdef PB_LSTM_TRACE
    PB_TRY(lstm_trace_buffer(1, &L.trace));
    PB_CUDA(cudaMemsetAsync(L.trace, 0, sizeof(uint64_t) * tc::lstm_trace_words(VT), st));
#endif
    static bool attr_set = false;
    if (!attr_set) {
        PB_CUDA(cudaFuncSetAttribute(tc::k_lstm_layer_q8, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::QSMEM_BYTES));
        attr_set = true;
    }
    for (int t0 = 0; t0 < VT; t0 = L.t1) {
        L.t0 = t0; L.t1 = std::min(t0 + steps, VT);
        tc::k_lstm_layer_q8<<<(unsigned) (2 * Mt), tc::LQ_THREADS, tc::QSMEM_BYTES, st>>>(L);
        N->launches++;
    }
    return PB_OK;
}

// linear_1 on int8 slices (mode 2): SELU(ydec W^T + b) from the decoder's h slices in T.ydec_q, all 33 steps read in place
// (slice k-tile tt * 8 + dir * 4 + unit / 64 is feature tt * 512 + dir * 256 + unit, linear_1's K order), into the fp16 tiles
// T.act_hi[0] / T.act_lo[0] that linear_2 reads (+ the optional fp32 copy y_f32 [B][512]).  One k_gemm_q8 launch.
static int variant_lin1_q8(pb_variant_net *N, int64_t B, float *y_f32, cudaStream_t st) {
    TcVariant &T = N->tc;
    const int64_t Mt = ceil_div(B, 128);
    tc::GemmQ G;
    memset(&G, 0, sizeof(G));
    G.a1 = T.ydec_q.as<int8_t>(); G.a0 = G.a1 + Mt * q_mt_bytes(); G.a_mt_stride = q_mt_bytes();
    G.w1 = T.lin1q.w1.as<int8_t>(); G.w0 = T.lin1q.w0.as<int8_t>();
    G.bias = T.lin[0].bias.as<float>(); G.col_scale = T.lin1q.col_scale.as<float>();
    G.y_hi = T.act_hi[0].as<bf16>(); G.y_lo = T.act_lo[0].as<bf16>(); G.y_f32 = y_f32;
    G.M = (int) B; G.N = 512; G.n_mt = (int) Mt; G.nkt = VT * 8;
    static bool attr_set = false;
    if (!attr_set) {
        PB_CUDA(cudaFuncSetAttribute(tc::k_gemm_q8, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::GQSMEM_BYTES));
        attr_set = true;
    }
    if (g_num_sms == 0) {
        int dev = 0;
        PB_CUDA(cudaGetDevice(&dev));
        PB_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
    }
    const int tiles = (int) Mt * (G.N / tc::QN);
    tc::k_gemm_q8<<<(unsigned) std::min(tiles, g_num_sms), tc::PG_THREADS, tc::GQSMEM_BYTES, st>>>(G);
    N->launches++;
    return PB_OK;
}

// scratch of one chunk of B candidates; the decoder's fp16 output tiles only for mode 1 (mode 2's linear_1 reads the slices)
static int variant_reserve_tc(TcVariant &T, int64_t B, int mode) {
    const int64_t Mt = ceil_div(B, 128), Bp = Mt * 128;
    const int64_t seq_tiles = Mt * VT * 16;                 // [mt][t][16 k-tiles] of a 512-feature sequence operand
    PB_TRY(T.img_op.reserve((size_t) (Mt * VT * TILE_ELEMS) * 2));
    PB_TRY(T.yenc_hi.reserve((size_t) (seq_tiles * TILE_ELEMS) * 2));
    PB_TRY(T.yenc_lo.reserve((size_t) (seq_tiles * TILE_ELEMS) * 2));
    if (mode == 1) {
        PB_TRY(T.ydec_hi.reserve((size_t) (seq_tiles * TILE_ELEMS) * 2));
        PB_TRY(T.ydec_lo.reserve((size_t) (seq_tiles * TILE_ELEMS) * 2));
    }
    PB_TRY(T.ydec_q.reserve((size_t) (2 * Mt * q_mt_bytes())));
    PB_TRY(T.c.reserve(sizeof(float) * 2 * VH * Bp));
    for (int i = 0; i < 2; i++) {
        PB_TRY(T.act_hi[i].reserve((size_t) (Mt * 16 * TILE_ELEMS) * 2));
        PB_TRY(T.act_lo[i].reserve((size_t) (Mt * 16 * TILE_ELEMS) * 2));
    }
    PB_TRY(T.final_f32.reserve(sizeof(float) * Bp * 512));
    return PB_OK;
}

// variant head: logits = W[3][512] x + b, softmax (simple_model.py:76-82); one warp per candidate.  With a record sink the
// warp also assembles the candidate's 84-byte prediction record (probabilities + the encoder's columns) in place, so the
// buffer a gather sends is produced by the network itself.
__global__ void k_variant_out(const float *__restrict__ x, const float *__restrict__ W, const float *__restrict__ b,
                              float *__restrict__ probs, int64_t n, pb::OutSink S) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int k = lane; k < 512; k += 32) {
        const float v = x[row * 512 + k];
        s0 = fmaf(v, __ldg(W + k), s0); s1 = fmaf(v, __ldg(W + 512 + k), s1); s2 = fmaf(v, __ldg(W + 1024 + k), s2);
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, d); s1 += __shfl_xor_sync(0xffffffffu, s1, d); s2 += __shfl_xor_sync(0xffffffffu, s2, d);
    }
    s0 += b[0]; s1 += b[1]; s2 += b[2];
    const float m = fmaxf(s0, fmaxf(s1, s2));
    const float e0 = expf(s0 - m), e1 = expf(s1 - m), e2 = expf(s2 - m);
    const float inv = 1.0f / (e0 + e1 + e2);
    if (lane == 0) { probs[row * 3 + 0] = e0 * inv; probs[row * 3 + 1] = e1 * inv; probs[row * 3 + 2] = e2 * inv; }
    if (S.records) {
        pb_pred_record_t *r = S.records + row;
        if (lane == 0) {
            r->probs[0] = e0 * inv; r->probs[1] = e1 * inv; r->probs[2] = e2 * inv;
            r->position = (int32_t) S.cols.positions[row];
            r->region = S.cols.region_of[row];
            r->depth = S.cols.depths[row]; r->freq = S.cols.freqs[row];
        } else {
            // lanes 1..31: two key bytes each (62 = 31 x 2); the key field starts at byte 22 of the 84-byte record
            const uint16_t kb = *reinterpret_cast<const uint16_t *>(S.cols.keys + row * PB_ALLELE_STRIDE + 2 * (lane - 1));
            *reinterpret_cast<uint16_t *>(r->key + 2 * (lane - 1)) = kb;
        }
    }
}

int variant_forward_tc(pb_variant_net *N, const int8_t *d_images, int64_t B, float *d_probs, float *d_hidden_dbg, cudaStream_t st,
                       const OutSink &sink) {
    TcVariant &T = N->tc;
    const int64_t Mt = ceil_div(B, 128), Bp = Mt * 128;
    PB_TRY(variant_reserve_tc(T, B, N->mode));

    tc::k_tc_pack_images<<<(unsigned) ceil_div(Bp * VT * 4, 256), 256, 0, st>>>(d_images, T.img_op.as<bf16>(), B, VT, 26);
    N->launches++;

    if (N->mode == 2) {
        // int8-slice decoder: the encoder runs its h-part hi only and hands the decoder its h as slices; lo_mask bits 0-2 do not
        // apply (set_lo_mask returns the network to mode 1)
        PB_TRY(variant_lstm_layer_tc(N, 0, B, true, false, true, nullptr, st, true));
        PB_TRY(variant_dec_q8(N, B, VT, d_hidden_dbg, st));
    } else {
        PB_TRY(variant_lstm_layer_tc(N, 0, B, true, T.lo_mask & 1, true, nullptr, st));
        PB_TRY(variant_lstm_layer_tc(N, 1, B, (T.lo_mask >> 1) & 1, (T.lo_mask >> 2) & 1, true, d_hidden_dbg, st));
    }
    // MLP head
    for (int i = 0; i < 5; i++) {
        if (i == 0 && N->mode == 2) {
            PB_TRY(variant_lin1_q8(N, B, nullptr, st));
            continue;
        }
        Args A;
        A.M = (int) B; A.N = 512;
        Dir D = empty_dir();
        if (i == 0) {
            D.seg[0].hi = T.ydec_hi.as<bf16>(); D.seg[0].lo = ((T.lo_mask >> 3) & 1) ? T.ydec_lo.as<bf16>() : nullptr;
            D.seg[0].mt_stride = (int64_t) VT * 16 * TILE_ELEMS; D.seg[0].nkt = VT * 16;
        } else {
            D.seg[0].hi = T.act_hi[(i - 1) & 1].as<bf16>(); D.seg[0].lo = ((T.lo_mask >> 4) & 1) ? T.act_lo[(i - 1) & 1].as<bf16>() : nullptr;
            D.seg[0].mt_stride = (int64_t) 16 * TILE_ELEMS; D.seg[0].nkt = 16;
        }
        D.w_hi = T.lin[i].w_hi.as<bf16>(); D.w_lo = T.lin[i].w_lo.as<bf16>(); D.w_nkt = T.lin[i].nkt;
        D.bias = T.lin[i].bias.as<float>();
        D.inv_scale = 1.f / T.lin[i].scale;
        D.y_hi = T.act_hi[i & 1].as<bf16>(); D.y_lo = T.act_lo[i & 1].as<bf16>(); D.y_mt_stride = (int64_t) 16 * TILE_ELEMS; D.y_kt0 = 0;
        if (i == 4) { D.y_f32 = T.final_f32.as<float>(); D.ldy = 512; }
        A.d[0] = D; A.d[1] = D;
        PB_TRY(launch_tc<tc::EPI_SELU>(A, (int) Mt, 4, 1, st));
        N->launches++;
    }
    k_variant_out<<<(unsigned) ceil_div(B, 8), 256, 0, st>>>(T.final_f32.as<float>(), N->out_w.as<float>(), N->out_b.as<float>(), d_probs, B, sink);
    N->launches++;
    PB_CUDA(cudaGetLastError());
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------- polish
constexpr int PH = 128, PWIN = 100;

// uint8 image window -> tiled operand [mt][100][1 k-tile] (values <= 254 are exact in bf16)
__global__ void k_tc_pack_polish(const uint8_t *__restrict__ img /* [B][1000][10] */, bf16 *__restrict__ op, int64_t B, int win_start) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;     // (row, t, kc)
    const int64_t total = ceil_div(B, 128) * 128 * PWIN * 4;
    if (i >= total) return;
    const int kc = (int) (i & 3);
    const int64_t rt = i >> 2;
    const int t = (int) (rt % PWIN);
    const int64_t row = rt / PWIN;
    uint32_t w[4] = {0, 0, 0, 0};
    if (row < B) {
#pragma unroll
        for (int e = 0; e < 8; e++) {
            const int k = kc * 8 + e;
            const float v = (k < 10) ? (float) img[(row * 1000 + win_start + t) * 10 + k] : 0.f;
            w[e >> 1] |= (uint32_t) tc::op_bits(v) << (16 * (e & 1));
        }
    }
    const int64_t o = ((row >> 7) * PWIN + t) * TILE_ELEMS + kc * 1024 + (row & 127) * 8;
    *reinterpret_cast<uint4 *>(op + o) = make_uint4(w[0], w[1], w[2], w[3]);
}

// hidden state [B][2][128] fp32 out of a sequence operand (fwd: time 99, bwd: time 0), for the debug read-back
__global__ void k_tc_unpack_hidden(const bf16 *__restrict__ y_hi, const bf16 *__restrict__ y_lo, float *__restrict__ out, int64_t B) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 2 * PH) return;
    const int j = (int) (i % PH);
    const int d = (int) ((i / PH) % 2);
    const int64_t b = i / (2 * PH);
    const int tt = d == 0 ? PWIN - 1 : 0;
    const int64_t o = (((b >> 7) * PWIN + tt) * 8 + d * 4 + (j >> 5)) * TILE_ELEMS + ((j & 31) >> 3) * 1024 + (b & 127) * 8 + (j & 7);
    out[i] = tc::op_val(reinterpret_cast<const uint16_t *>(y_hi)[o]) + tc::op_val(reinterpret_cast<const uint16_t *>(y_lo)[o]);
}
// dense1 (256 -> 5) + softmax + window accumulate straight from the decoder's tiled output operand
// (predict_distributed_cpu.py:62-81): one thread per (image row, time step); lanes = consecutive rows of a row tile, so
// every 16-byte operand load is coalesced; no fp32 copy of the decoder output is ever written.
__global__ void __launch_bounds__(128) k_polish_dense_tiles(const bf16 *__restrict__ y_hi, const bf16 *__restrict__ y_lo,
                                                            const float *__restrict__ W /* [5][256] */, const float *__restrict__ bias,
                                                            float *__restrict__ acc /* [B][1000][5] */, int64_t B, int win_start) {
    __shared__ float sW[5 * 256];
    for (int i = threadIdx.x; i < 5 * 256; i += 128) sW[i] = W[i];
    __syncthreads();
    const int64_t mt = blockIdx.x / PWIN;
    const int t = (int) (blockIdx.x % PWIN);
    const int r128 = threadIdx.x;
    const int64_t row = mt * 128 + r128;
    if (row >= B) return;
    float s[5] = {bias[0], bias[1], bias[2], bias[3], bias[4]};
    const int64_t tile0 = (mt * PWIN + t) * 8;
#pragma unroll 2
    for (int kt = 0; kt < 8; kt++) {
#pragma unroll
        for (int kc = 0; kc < 4; kc++) {
            const int64_t o = (tile0 + kt) * TILE_ELEMS + kc * 1024 + r128 * 8;
            const uint4 h = *reinterpret_cast<const uint4 *>(y_hi + o), l = *reinterpret_cast<const uint4 *>(y_lo + o);
            const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const float v = tc::op_val(hw[e >> 1] >> (16 * (e & 1))) + tc::op_val(lw[e >> 1] >> (16 * (e & 1)));
                const int f = kt * 32 + kc * 8 + e;
#pragma unroll
                for (int c = 0; c < 5; c++) s[c] = fmaf(v, sW[c * 256 + f], s[c]);
            }
        }
    }
    float m = s[0];
#pragma unroll
    for (int c = 1; c < 5; c++) m = fmaxf(m, s[c]);
    float e[5], sum = 0.f;
#pragma unroll
    for (int c = 0; c < 5; c++) { e[c] = expf(s[c] - m); sum += e[c]; }
    float *dst = acc + (row * 1000 + win_start + t) * 5;
#pragma unroll
    for (int c = 0; c < 5; c++) dst[c] += e[c] / sum;
}

// one bidirectional GRU layer over the 100 steps of a window: ONE launch of k_gru_layer, one CTA per (direction, row tile).
//   x operand: [mt][100][xkt] tiles (hi, lo or hi only); h0 of direction d: 4 k-tiles per row tile at h0_hi[d] +
//   mt * h0_mt_stride (the state of another sequence operand, or the zero operand with stride 0).  lo_x / lo_h: the
//   a_lo x w_hi product of the x-part / h-part runs.
static int gru_layer_tc(pb_polish_net *N, int layer, const bf16 *x_hi, const bf16 *x_lo, const bf16 *const h0_hi[2],
                        const bf16 *const h0_lo[2], int64_t h0_mt_stride, bool lo_x, bool lo_h, bf16 *y_hi, bf16 *y_lo, int64_t B,
                        cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        PB_CUDA(cudaFuncSetAttribute(tc::k_gru_layer, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::PSMEM_BYTES));
        attr_set = true;
    }
    TcRnn *W = layer == 0 ? N->tc.enc : N->tc.dec;
    const int xkt = layer == 0 ? 1 : 8;
    const int64_t Mt = ceil_div(B, 128);
    tc::GruWin G;
    G.x_hi = x_hi; G.x_lo = x_lo; G.x_kt = xkt;
    for (int d = 0; d < 2; d++) {
        G.h0_hi[d] = h0_hi[d]; G.h0_lo[d] = h0_lo[d];
        G.w_hi[d] = W[d].w_hi.as<bf16>(); G.w_lo[d] = W[d].w_lo.as<bf16>();
        G.bias[d] = W[d].bias.as<float>();
        G.inv_scale[d] = 1.f / W[d].scale;
        if (W[d].nkt_x != xkt || W[d].nkt_h != 4) { set_error("gru_layer_tc: weight / operand k-tile mismatch"); return PB_ERR_STATE; }
    }
    G.h0_mt_stride = h0_mt_stride;
    G.y_hi = y_hi; G.y_lo = y_lo;
    G.M = (int) B; G.n_mt = (int) Mt; G.T = PWIN;
    G.lo_x = lo_x; G.lo_h = lo_h;
    tc::k_gru_layer<<<(unsigned) (2 * Mt), tc::PG_THREADS, tc::PSMEM_BYTES, st>>>(G);
    PB_CUDA(cudaGetLastError());
    N->launches++;
    return PB_OK;
}

// scratch of one chunk of B images
static int polish_reserve_tc(TcPolish &T, int64_t B) {
    const int64_t Mt = ceil_div(B, 128);
    const int64_t seq = Mt * PWIN * 8 * TILE_ELEMS;
    PB_TRY(T.img_op.reserve((size_t) (Mt * PWIN * TILE_ELEMS) * 2));
    PB_TRY(T.yenc_hi.reserve((size_t) seq * 2)); PB_TRY(T.yenc_lo.reserve((size_t) seq * 2));
    PB_TRY(T.ydec_hi.reserve((size_t) seq * 2)); PB_TRY(T.ydec_lo.reserve((size_t) seq * 2));
    PB_TRY(T.zero.reserve((size_t) 4 * TILE_ELEMS * 2));
    return PB_OK;
}

int polish_forward_tc(pb_polish_net *N, const uint8_t *d_images, int64_t B, int64_t n_total, int64_t b0, float *d_hidden_dbg,
                      cudaStream_t st) {
    TcPolish &T = N->tc;
    const int64_t Mt = ceil_div(B, 128);
    const int64_t ystride = (int64_t) PWIN * 8 * TILE_ELEMS;
    PB_TRY(polish_reserve_tc(T, B));
    PB_CUDA(cudaMemsetAsync(T.zero.p, 0, (size_t) 4 * TILE_ELEMS * 2, st));
    // the final state of a sequence operand: fwd at time 99, bwd at time 0
    auto final_state = [](const bf16 *y, int d) { return y + ((int64_t) (d == 0 ? PWIN - 1 : 0) * 8 + d * 4) * TILE_ELEMS; };
    const bf16 *zero[2] = {T.zero.as<bf16>(), T.zero.as<bf16>()};
    const bf16 *enc_hi[2] = {final_state(T.yenc_hi.as<bf16>(), 0), final_state(T.yenc_hi.as<bf16>(), 1)};
    const bf16 *enc_lo[2] = {final_state(T.yenc_lo.as<bf16>(), 0), final_state(T.yenc_lo.as<bf16>(), 1)};
    const bf16 *dec_hi[2] = {final_state(T.ydec_hi.as<bf16>(), 0), final_state(T.ydec_hi.as<bf16>(), 1)};
    const bf16 *dec_lo[2] = {final_state(T.ydec_lo.as<bf16>(), 0), final_state(T.ydec_lo.as<bf16>(), 1)};
    for (int w = 0; w < 19; w++) {
        const int i = w * 50;
        k_tc_pack_polish<<<(unsigned) ceil_div(Mt * 128 * PWIN * 4, 256), 256, 0, st>>>(d_images, T.img_op.as<bf16>(), B, i);
        N->launches++;
        // encoder: h0 = carried state (decoder's final state of the previous window, zeros for the first); uint8 images are exact
        PB_TRY(gru_layer_tc(N, 0, T.img_op.as<bf16>(), nullptr, w == 0 ? zero : dec_hi, w == 0 ? zero : dec_lo, w == 0 ? 0 : ystride,
                            true, T.lo_mask & 1, T.yenc_hi.as<bf16>(), T.yenc_lo.as<bf16>(), B, st));
        // decoder: h0 = encoder's final state
        PB_TRY(gru_layer_tc(N, 1, T.yenc_hi.as<bf16>(), T.yenc_lo.as<bf16>(), enc_hi, enc_lo, ystride, (T.lo_mask >> 1) & 1,
                            (T.lo_mask >> 2) & 1, T.ydec_hi.as<bf16>(), T.ydec_lo.as<bf16>(), B, st));
        if (d_hidden_dbg) {
            k_tc_unpack_hidden<<<(unsigned) ceil_div(B * 2 * PH, 256), 256, 0, st>>>(T.ydec_hi.as<bf16>(), T.ydec_lo.as<bf16>(),
                                                                                    d_hidden_dbg + ((int64_t) w * n_total + b0) * 2 * PH, B);
            N->launches++;
        }
        k_polish_dense_tiles<<<(unsigned) (Mt * PWIN), 128, 0, st>>>(T.ydec_hi.as<bf16>(), T.ydec_lo.as<bf16>(), N->dW.as<float>(), N->dB.as<float>(),
                                                                    N->acc.as<float>(), B, i);
        N->launches++;
    }
    PB_CUDA(cudaGetLastError());
    return PB_OK;
}

}  // namespace pb

// ------------------------------------------------------------------------------------------------- self tests
// Diagnostic entry points that run the production launch code on inputs given by the caller (include/pepper_b200.h).
// `poison`: every operand buffer the launch reads or writes is first filled with 0xFFFF (fp16 NaN), and the padding rows
// of host-tiled inputs are NaN, so a padding row or k column that reaches a valid output shows up as a non-finite value.
namespace {
struct Scratch {                       // device buffers released on every return path
    DevBuf b[8];
    ~Scratch() { for (auto &x : b) x.release(); }
};
void poison_rows(std::vector<uint16_t> &t, int64_t rows, int64_t rows_p, int64_t Kp) {
    for (int64_t r = rows; r < rows_p; r++)
        for (int64_t k = 0; k < Kp; k++) t[(size_t) tiled_index(r, k, Kp / 32, 128)] = 0xffffu;
}
int need_device() {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) { set_error("no CUDA device: libpepper_b200 has no CPU fallback"); return PB_ERR_CUDA; }
    return PB_OK;
}
int fill_nan(DevBuf &b) {
    PB_CUDA(cudaMemset(b.p, 0xff, b.cap));
    return PB_OK;
}
}  // namespace

// fp32 [rows][K] -> the hi / lo tile images of tile_matrix (the packing of every host-tiled operand and weight).
// tile_rows 128 (A operands) or 256 (weights); hi / lo hold ceil(rows / tile_rows) * tile_rows * ceil(K / 32) * 32 elements.
extern "C" int pb_test_tc_split_tiles(int64_t rows, int64_t K, int tile_rows, const float *src, uint16_t *hi, uint16_t *lo) {
    if (rows <= 0 || K <= 0 || (tile_rows != 128 && tile_rows != 256) || !src || !hi || !lo) { set_error("pb_test_tc_split_tiles: bad argument"); return PB_ERR_ARG; }
    const int64_t rows_p = (rows + tile_rows - 1) / tile_rows * tile_rows, Kp = (K + 31) / 32 * 32;
    std::vector<uint16_t> h, l;
    tile_matrix(src, rows, K, rows_p, Kp, h, l, tile_rows);
    memcpy(hi, h.data(), h.size() * 2);
    memcpy(lo, l.data(), l.size() * 2);
    return PB_OK;
}

// Y = epi(A W^T + bias) through k_tc_gemm_p: A = [A0 | A1] as two K segments (K1 == 0: one), each with its own lo operand
// flag; W [N][K0 + K1] packed and scaled as a linear layer; optional fp32 output [M][N] and output tiles [Mt][N / 32][4096].
extern "C" int pb_test_tc_gemm_ex(int M, int N, int epi, int K0, const float *h_A0, int lo0, int K1, const float *h_A1, int lo1,
                                  const float *h_W, const float *h_bias, int max_ctas, int poison, float *h_out, uint16_t *h_y_hi,
                                  uint16_t *h_y_lo) {
    if (M <= 0 || N <= 0 || N % 256 || K0 <= 0 || K0 % 32 || K1 < 0 || K1 % 32 || (K1 && !h_A1) || !h_A0 || !h_W || !h_bias ||
        (epi != tc::EPI_BIAS && epi != tc::EPI_SELU) || (!h_y_hi) != (!h_y_lo)) {
        set_error("pb_test_tc_gemm_ex: N %% 256 and K %% 32 must be 0, epi 0 (bias) or 1 (SELU)");
        return PB_ERR_ARG;
    }
    PB_TRY(need_device());
    const int64_t Mt = ceil_div(M, 128);
    Scratch S;
    DevBuf &a0hi = S.b[0], &a0lo = S.b[1], &a1hi = S.b[2], &a1lo = S.b[3], &dout = S.b[5], &yhi = S.b[6], &ylo = S.b[7];
    std::vector<uint16_t> hi, lo;
    tile_matrix(h_A0, M, K0, Mt * 128, K0, hi, lo);
    if (poison) { poison_rows(hi, M, Mt * 128, K0); poison_rows(lo, M, Mt * 128, K0); }
    PB_TRY(upload_tiles(a0hi, a0lo, hi, lo));
    if (K1) {
        tile_matrix(h_A1, M, K1, Mt * 128, K1, hi, lo);
        if (poison) { poison_rows(hi, M, Mt * 128, K1); poison_rows(lo, M, Mt * 128, K1); }
        PB_TRY(upload_tiles(a1hi, a1lo, hi, lo));
    }
    TcLin W;
    int rc = tc_upload_lin(W, h_W, h_bias, N, K0 + K1);
    Args A;
    A.M = M; A.N = N;
    Dir D = empty_dir();
    D.seg[0].hi = a0hi.as<bf16>(); D.seg[0].lo = lo0 ? a0lo.as<bf16>() : nullptr; D.seg[0].mt_stride = (int64_t) (K0 / 32) * TILE_ELEMS; D.seg[0].nkt = K0 / 32;
    if (K1) { D.seg[1].hi = a1hi.as<bf16>(); D.seg[1].lo = lo1 ? a1lo.as<bf16>() : nullptr; D.seg[1].mt_stride = (int64_t) (K1 / 32) * TILE_ELEMS; D.seg[1].nkt = K1 / 32; }
    D.w_hi = W.w_hi.as<bf16>(); D.w_lo = W.w_lo.as<bf16>(); D.w_nkt = W.nkt;
    D.inv_scale = 1.f / W.scale;
    D.bias = W.bias.as<float>();
    if (rc == PB_OK && h_out) rc = dout.reserve(sizeof(float) * (size_t) M * N);
    if (rc == PB_OK && h_y_hi) rc = yhi.reserve((size_t) (Mt * (N / 32) * TILE_ELEMS) * 2);
    if (rc == PB_OK && h_y_hi) rc = ylo.reserve((size_t) (Mt * (N / 32) * TILE_ELEMS) * 2);
    if (rc == PB_OK) {
        cudaError_t e = h_out ? cudaMemset(dout.p, poison ? 0xff : 0, dout.cap) : cudaSuccess;
        if (e == cudaSuccess && h_y_hi) e = cudaMemset(yhi.p, poison ? 0xff : 0, yhi.cap);
        if (e == cudaSuccess && h_y_hi) e = cudaMemset(ylo.p, poison ? 0xff : 0, ylo.cap);
        if (e != cudaSuccess) { set_error("pb_test_tc_gemm_ex: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    }
    if (rc == PB_OK) {
        if (h_out) { D.y_f32 = dout.as<float>(); D.ldy = N; }
        if (h_y_hi) { D.y_hi = yhi.as<bf16>(); D.y_lo = ylo.as<bf16>(); D.y_mt_stride = (int64_t) (N / 32) * TILE_ELEMS; D.y_kt0 = 0; }
        A.d[0] = D; A.d[1] = D;
        rc = epi == tc::EPI_SELU ? launch_tc<tc::EPI_SELU>(A, (int) Mt, N / 128, 1, 0, max_ctas) : launch_tc<tc::EPI_BIAS>(A, (int) Mt, N / 128, 1, 0, max_ctas);
    }
    if (rc == PB_OK) {
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e == cudaSuccess && h_out) e = cudaMemcpy(h_out, dout.p, sizeof(float) * (size_t) M * N, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess && h_y_hi) e = cudaMemcpy(h_y_hi, yhi.p, (size_t) (Mt * (N / 32) * TILE_ELEMS) * 2, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess && h_y_hi) e = cudaMemcpy(h_y_lo, ylo.p, (size_t) (Mt * (N / 32) * TILE_ELEMS) * 2, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { set_error("pb_test_tc_gemm_ex: %s", cudaGetErrorString(e)); rc = PB_ERR_CUDA; }
    }
    W.w_hi.release(); W.w_lo.release(); W.bias.release();
    return rc;
}

// C[M][N] = A[M][K] W[N][K]^T + bias through the wgmma kernel (EPI_BIAS, fp32 output).  N % 256 == 0, K % 32 == 0.
extern "C" int pb_test_tc_gemm(int M, int N, int K, const float *h_A, const float *h_W, const float *h_bias, float *h_out) {
    return pb_test_tc_gemm_ex(M, N, tc::EPI_BIAS, K, h_A, 1, 0, nullptr, 0, h_W, h_bias, 0, 0, h_out, nullptr, nullptr);
}

// The cell state the last variant LSTM layer left in T.c (tc::c_index per direction) as c_final [2][256][M].
static int read_c_final(TcVariant &T, int M, float *h_c_final) {
    const int64_t per_dir = ceil_div(M, 128) * 128 * VH;
    std::vector<float> c((size_t) (2 * per_dir));
    PB_CUDA(cudaMemcpy(c.data(), T.c.p, sizeof(float) * c.size(), cudaMemcpyDeviceToHost));
    for (int d = 0; d < 2; d++)
        for (int u = 0; u < VH; u++)
            for (int r = 0; r < M; r++) h_c_final[((size_t) d * VH + u) * M + r] = c[d * per_dir + tc::c_index(u, r)];
    return PB_OK;
}

// One LSTM layer of the variant network (variant_lstm_layer_tc, the forward pass's own launch code) with the network's packed
// weights.  x: int8 images [M][33][26] (layer 0) or fp32 [M][33][512] (layer 1, tiled like every host operand).  Outputs
// (each may be NULL): y_f32 [M][33][512]; the output sequence tiles [Mt][33][16][4096] hi / lo; the final cell state
// c_final [2][256][M].
extern "C" int pb_test_variant_lstm_layer(pb_variant_net_t *net, int layer, int M, const void *h_x, int lo_x, int lo_h, int persist,
                                          int poison, float *h_y_f32, uint16_t *h_y_hi, uint16_t *h_y_lo, float *h_c_final) {
    if (!net || (layer != 0 && layer != 1) || M <= 0 || !h_x || (!h_y_hi) != (!h_y_lo)) {
        set_error("pb_test_variant_lstm_layer: bad argument");
        return PB_ERR_ARG;
    }
    PB_CUDA(cudaSetDevice(net->device));
    TcVariant &T = net->tc;
    const int64_t Mt = ceil_div(M, 128), Bp = Mt * 128, seq = Mt * VT * 16 * TILE_ELEMS;
    PB_TRY(variant_reserve_tc(T, M, 1));
    if (poison) {
        DevBuf *bufs[] = {&T.img_op, &T.yenc_hi, &T.yenc_lo, &T.ydec_hi, &T.ydec_lo, &T.c};
        for (auto *b : bufs) PB_TRY(fill_nan(*b));
    }
    Scratch S;
    if (layer == 0) {
        PB_TRY(S.b[0].reserve((size_t) M * VT * 26));
        PB_CUDA(cudaMemcpy(S.b[0].p, h_x, (size_t) M * VT * 26, cudaMemcpyHostToDevice));
        tc::k_tc_pack_images<<<(unsigned) ceil_div(Bp * VT * 4, 256), 256, 0>>>(S.b[0].as<int8_t>(), T.img_op.as<bf16>(), M, VT, 26);
    } else {
        std::vector<uint16_t> hi, lo;
        tile_matrix(static_cast<const float *>(h_x), M, VT * 512, Bp, VT * 512, hi, lo);
        if (poison) { poison_rows(hi, M, Bp, VT * 512); poison_rows(lo, M, Bp, VT * 512); }
        PB_CUDA(cudaMemcpy(T.yenc_hi.p, hi.data(), hi.size() * 2, cudaMemcpyHostToDevice));
        PB_CUDA(cudaMemcpy(T.yenc_lo.p, lo.data(), lo.size() * 2, cudaMemcpyHostToDevice));
    }
    if (h_y_f32) {
        PB_TRY(S.b[1].reserve(sizeof(float) * (size_t) M * VT * 512));
        PB_CUDA(cudaMemset(S.b[1].p, poison ? 0xff : 0, S.b[1].cap));
    }
    PB_TRY(variant_lstm_layer_tc(net, layer, M, lo_x != 0, lo_h != 0, persist != 0, h_y_f32 ? S.b[1].as<float>() : nullptr, 0));
    PB_CUDA(cudaGetLastError());
    PB_CUDA(cudaDeviceSynchronize());
    if (h_y_f32) PB_CUDA(cudaMemcpy(h_y_f32, S.b[1].p, sizeof(float) * (size_t) M * VT * 512, cudaMemcpyDeviceToHost));
    if (h_y_hi) {
        PB_CUDA(cudaMemcpy(h_y_hi, (layer == 0 ? T.yenc_hi : T.ydec_hi).p, (size_t) seq * 2, cudaMemcpyDeviceToHost));
        PB_CUDA(cudaMemcpy(h_y_lo, (layer == 0 ? T.yenc_lo : T.ydec_lo).p, (size_t) seq * 2, cudaMemcpyDeviceToHost));
    }
    if (h_c_final) PB_TRY(read_c_final(T, M, h_c_final));
    return PB_OK;
}

// The encoder layer of mode 2 (the forward pass's own launch code): h as the decoder's int8 x slices.  h_x: int8 images
// [M][33][26].  h_q: the slice images as the layer leaves them in T.yenc_lo, int8 [2][Mt][33][8][128][64] (slice 1, then
// slice 0; tc_gemm.cuh QSeq layout).  poison: that buffer is first filled with 0xff bytes, which padding rows keep.
extern "C" int pb_test_variant_enc_q8(pb_variant_net_t *net, int M, const int8_t *h_x, int poison, int8_t *h_q) {
    if (!net || M <= 0 || !h_x || !h_q) { set_error("pb_test_variant_enc_q8: bad argument"); return PB_ERR_ARG; }
    PB_CUDA(cudaSetDevice(net->device));
    TcVariant &T = net->tc;
    const int64_t Mt = ceil_div(M, 128), Bp = Mt * 128;
    PB_TRY(variant_reserve_tc(T, M, 2));
    if (poison) PB_TRY(fill_nan(T.yenc_lo));
    Scratch S;
    PB_TRY(S.b[0].reserve((size_t) M * VT * 26));
    PB_CUDA(cudaMemcpy(S.b[0].p, h_x, (size_t) M * VT * 26, cudaMemcpyHostToDevice));
    tc::k_tc_pack_images<<<(unsigned) ceil_div(Bp * VT * 4, 256), 256, 0>>>(S.b[0].as<int8_t>(), T.img_op.as<bf16>(), M, VT, 26);
    PB_TRY(variant_lstm_layer_tc(net, 0, M, true, false, true, nullptr, 0, true));
    PB_CUDA(cudaGetLastError());
    PB_CUDA(cudaDeviceSynchronize());
    PB_CUDA(cudaMemcpy(h_q, T.yenc_lo.p, (size_t) (2 * Mt * q_mt_bytes()), cudaMemcpyDeviceToHost));
    return PB_OK;
}

// The int8-slice decoder layer (variant_dec_q8, the forward pass's own launch code) on host-quantized input slices.  persist:
// 1 one launch, 0 one launch per step, k >= 2 launches of k steps.
extern "C" int pb_test_variant_lstm_q8(pb_variant_net_t *net, int M, const float *h_x, int persist, int poison, float *h_y_f32, int8_t *h_q,
                                       float *h_c_final) {
    if (!net || M <= 0 || !h_x || persist < 0) { set_error("pb_test_variant_lstm_q8: bad argument"); return PB_ERR_ARG; }
    PB_CUDA(cudaSetDevice(net->device));
    TcVariant &T = net->tc;
    const int64_t Mt = ceil_div(M, 128), qbytes = Mt * q_mt_bytes();
    PB_TRY(variant_reserve_tc(T, M, 2));
    if (poison) {
        DevBuf *bufs[] = {&T.yenc_lo, &T.ydec_q, &T.c};
        for (auto *b : bufs) PB_TRY(fill_nan(*b));
    }
    // the encoder's quantization (tc_gemm.cuh qsplit2): rint(fp32(clamp(x, -1, 1) * 32512))
    std::vector<int8_t> q(2 * qbytes, poison ? (int8_t) -1 : (int8_t) 0);
    for (int64_t r = 0; r < M; r++)
        for (int64_t k = 0; k < VT * 512; k++) {
            const float v = std::min(std::max(h_x[r * VT * 512 + k], -1.f), 1.f) * tc::QSCALE;
            const int64_t o = qtiled_index(r, k, VT * 8);
            qsplit(v, q[o], q[qbytes + o]);
        }
    PB_CUDA(cudaMemcpy(T.yenc_lo.p, q.data(), q.size(), cudaMemcpyHostToDevice));
    Scratch S;
    // y_f32 with room for the padding rows too: under poison they must come back as the 0xff bytes they started as
    const size_t y_rows = (size_t) (poison ? Mt * 128 : M), y_row_bytes = sizeof(float) * VT * 512;
    if (h_y_f32) {
        PB_TRY(S.b[0].reserve(y_rows * y_row_bytes));
        PB_CUDA(cudaMemset(S.b[0].p, poison ? 0xff : 0, S.b[0].cap));
    }
    PB_TRY(variant_dec_q8(net, M, persist == 0 ? 1 : persist == 1 ? VT : persist, h_y_f32 ? S.b[0].as<float>() : nullptr, 0));
    PB_CUDA(cudaGetLastError());
    PB_CUDA(cudaDeviceSynchronize());
    if (h_y_f32) {
        PB_CUDA(cudaMemcpy(h_y_f32, S.b[0].p, (size_t) M * y_row_bytes, cudaMemcpyDeviceToHost));
        if (y_rows > (size_t) M) {
            std::vector<uint8_t> pad((y_rows - M) * y_row_bytes);
            PB_CUDA(cudaMemcpy(pad.data(), S.b[0].as<uint8_t>() + (size_t) M * y_row_bytes, pad.size(), cudaMemcpyDeviceToHost));
            if (std::any_of(pad.begin(), pad.end(), [](uint8_t v) { return v != 0xff; })) {
                set_error("pb_test_variant_lstm_q8: a padding row of y_f32 was written");
                return PB_ERR_STATE;
            }
        }
    }
    if (h_q) PB_CUDA(cudaMemcpy(h_q, T.ydec_q.p, (size_t) (2 * qbytes), cudaMemcpyDeviceToHost));
    if (h_c_final) PB_TRY(read_c_final(T, M, h_c_final));
    return PB_OK;
}

// linear_1 of mode 2 (variant_lin1_q8, the forward pass's own launch code) on host-given slices of the decoder's h.
extern "C" int pb_test_variant_head_q8(pb_variant_net_t *net, int M, const int8_t *h_q, int poison, float *h_out, uint16_t *h_y_hi,
                                       uint16_t *h_y_lo) {
    if (!net || M <= 0 || !h_q || (!h_y_hi) != (!h_y_lo)) { set_error("pb_test_variant_head_q8: bad argument"); return PB_ERR_ARG; }
    PB_CUDA(cudaSetDevice(net->device));
    TcVariant &T = net->tc;
    const int64_t Mt = ceil_div(M, 128), qbytes = Mt * q_mt_bytes(), K = VT * 512, act = Mt * 16 * TILE_ELEMS;
    PB_TRY(variant_reserve_tc(T, M, 2));
    if (poison) {
        DevBuf *bufs[] = {&T.act_hi[0], &T.act_lo[0]};
        for (auto *b : bufs) PB_TRY(fill_nan(*b));
    }
    std::vector<int8_t> q(2 * qbytes, poison ? (int8_t) -1 : (int8_t) 0);
    for (int s = 0; s < 2; s++)
        for (int64_t r = 0; r < M; r++)
            for (int64_t k = 0; k < K; k++) q[s * qbytes + qtiled_index(r, k, VT * 8)] = h_q[(s * (int64_t) M + r) * K + k];
    PB_CUDA(cudaMemcpy(T.ydec_q.p, q.data(), q.size(), cudaMemcpyHostToDevice));
    Scratch S;
    if (h_out) {
        PB_TRY(S.b[0].reserve(sizeof(float) * (size_t) M * 512));
        PB_CUDA(cudaMemset(S.b[0].p, poison ? 0xff : 0, S.b[0].cap));
    }
    PB_TRY(variant_lin1_q8(net, M, h_out ? S.b[0].as<float>() : nullptr, 0));
    PB_CUDA(cudaGetLastError());
    PB_CUDA(cudaDeviceSynchronize());
    if (h_out) PB_CUDA(cudaMemcpy(h_out, S.b[0].p, sizeof(float) * (size_t) M * 512, cudaMemcpyDeviceToHost));
    if (h_y_hi) {
        PB_CUDA(cudaMemcpy(h_y_hi, T.act_hi[0].p, (size_t) act * 2, cudaMemcpyDeviceToHost));
        PB_CUDA(cudaMemcpy(h_y_lo, T.act_lo[0].p, (size_t) act * 2, cudaMemcpyDeviceToHost));
    }
    return PB_OK;
}

// The host packing of a weight matrix on int8 slices (pack_q8).  No GPU needed.
extern "C" int pb_test_q8_pack(int N, int K, const float *h_W, int a_quant, int8_t *h_w1, int8_t *h_w0, float *h_col_scale,
                               double *h_row_err) {
    if (N <= 0 || K <= 0 || N % tc::QN || K % tc::QK || !h_W || !h_w1 || !h_w0 || !h_col_scale || !h_row_err) {
        set_error("pb_test_q8_pack: N %% 128 and K %% 64 must be 0");
        return PB_ERR_ARG;
    }
    std::vector<int8_t> w1, w0;
    std::vector<float> cs;
    std::vector<double> err;
    pack_q8(h_W, N, K, a_quant != 0, w1, w0, cs, err);
    memcpy(h_w1, w1.data(), w1.size());
    memcpy(h_w0, w0.data(), w0.size());
    memcpy(h_col_scale, cs.data(), sizeof(float) * N);
    memcpy(h_row_err, err.data(), sizeof(double) * N);
    return PB_OK;
}

// One GRU layer of the polish network over one 100-step window (gru_layer_tc) with the network's packed weights.
// x: uint8 images [M][100][10] (layer 0) or fp32 [M][100][256] (layer 1); h0: [2][M][128] fp32 or NULL (zero state).
// Output: the sequence tiles [Mt][100][8][4096] hi / lo.
extern "C" int pb_test_polish_gru_layer(pb_polish_net_t *net, int layer, int M, const void *h_x, const float *h_h0, int lo_x, int lo_h,
                                        int poison, uint16_t *h_y_hi, uint16_t *h_y_lo) {
    if (!net || (layer != 0 && layer != 1) || M <= 0 || !h_x || !h_y_hi || !h_y_lo) {
        set_error("pb_test_polish_gru_layer: bad argument");
        return PB_ERR_ARG;
    }
    PB_CUDA(cudaSetDevice(net->device));
    TcPolish &T = net->tc;
    const int64_t Mt = ceil_div(M, 128), Bp = Mt * 128, seq = Mt * PWIN * 8 * TILE_ELEMS;
    PB_TRY(polish_reserve_tc(T, M));
    if (poison) {
        DevBuf *bufs[] = {&T.img_op, &T.yenc_hi, &T.yenc_lo, &T.ydec_hi, &T.ydec_lo};
        for (auto *b : bufs) PB_TRY(fill_nan(*b));
    }
    PB_CUDA(cudaMemset(T.zero.p, 0, (size_t) 4 * TILE_ELEMS * 2));
    Scratch S;
    if (layer == 0) {
        // the pack kernel reads windows of a [M][1000][10] image: the window at 0 holds the input
        PB_TRY(S.b[0].reserve((size_t) M * 1000 * 10));
        PB_CUDA(cudaMemset(S.b[0].p, 0, (size_t) M * 1000 * 10));
        PB_CUDA(cudaMemcpy2D(S.b[0].p, 1000 * 10, h_x, PWIN * 10, PWIN * 10, M, cudaMemcpyHostToDevice));
        k_tc_pack_polish<<<(unsigned) ceil_div(Bp * PWIN * 4, 256), 256, 0>>>(S.b[0].as<uint8_t>(), T.img_op.as<bf16>(), M, 0);
    } else {
        std::vector<uint16_t> hi, lo;
        tile_matrix(static_cast<const float *>(h_x), M, PWIN * 256, Bp, PWIN * 256, hi, lo);
        if (poison) { poison_rows(hi, M, Bp, PWIN * 256); poison_rows(lo, M, Bp, PWIN * 256); }
        PB_CUDA(cudaMemcpy(T.yenc_hi.p, hi.data(), hi.size() * 2, cudaMemcpyHostToDevice));
        PB_CUDA(cudaMemcpy(T.yenc_lo.p, lo.data(), lo.size() * 2, cudaMemcpyHostToDevice));
    }
    const bf16 *h0_hi[2] = {T.zero.as<bf16>(), T.zero.as<bf16>()}, *h0_lo[2] = {T.zero.as<bf16>(), T.zero.as<bf16>()};
    int64_t h0_stride = 0;
    if (h_h0) {
        const int64_t per_dir = Mt * 4 * TILE_ELEMS;
        PB_TRY(S.b[1].reserve((size_t) (2 * per_dir) * 2));
        PB_TRY(S.b[2].reserve((size_t) (2 * per_dir) * 2));
        for (int d = 0; d < 2; d++) {
            std::vector<uint16_t> hi, lo;
            tile_matrix(h_h0 + (size_t) d * M * PH, M, PH, Bp, PH, hi, lo);
            if (poison) { poison_rows(hi, M, Bp, PH); poison_rows(lo, M, Bp, PH); }
            PB_CUDA(cudaMemcpy(S.b[1].as<bf16>() + d * per_dir, hi.data(), hi.size() * 2, cudaMemcpyHostToDevice));
            PB_CUDA(cudaMemcpy(S.b[2].as<bf16>() + d * per_dir, lo.data(), lo.size() * 2, cudaMemcpyHostToDevice));
            h0_hi[d] = S.b[1].as<bf16>() + d * per_dir; h0_lo[d] = S.b[2].as<bf16>() + d * per_dir;
        }
        h0_stride = 4 * TILE_ELEMS;
    }
    const bf16 *x_hi = layer == 0 ? T.img_op.as<bf16>() : T.yenc_hi.as<bf16>();
    const bf16 *x_lo = layer == 0 ? nullptr : T.yenc_lo.as<bf16>();
    bf16 *y_hi = layer == 0 ? T.yenc_hi.as<bf16>() : T.ydec_hi.as<bf16>();
    bf16 *y_lo = layer == 0 ? T.yenc_lo.as<bf16>() : T.ydec_lo.as<bf16>();
    PB_TRY(gru_layer_tc(net, layer, x_hi, x_lo, h0_hi, h0_lo, h0_stride, lo_x != 0, lo_h != 0, y_hi, y_lo, M, 0));
    PB_CUDA(cudaDeviceSynchronize());
    PB_CUDA(cudaMemcpy(h_y_hi, y_hi, (size_t) seq * 2, cudaMemcpyDeviceToHost));
    PB_CUDA(cudaMemcpy(h_y_lo, y_lo, (size_t) seq * 2, cudaMemcpyDeviceToHost));
    return PB_OK;
}
