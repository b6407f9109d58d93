// wgmma GEMM with fused LSTM / GRU / SELU epilogues for sm_90a (H100).
//
//   D[128 x 256] (fp32, registers)  +=  A[128 x 32] (16-bit, smem)  x  B[256 x 32]^T (16-bit, smem)      per k-tile
//
// Precision comes from a hi/lo split of BOTH operands (22 significant bits) and three tensor-core products per k-tile
// accumulated into the same fp32 tile:  a*w ~= a_hi*w_hi + a_hi*w_lo + a_lo*w_hi.  This is not fp32-equivalent: measured on
// H100 the wgmma accumulation error grows about linearly with K, and a layer's error against exact float64 is 2-5x that of a
// float32 CPU layer (tests/test_tc_layers_gpu.py).  Each packed weight matrix is scaled by a
// power of two s (max |s W| in (2^14, 2^15]) so that w_lo stays out of the fp16 subnormals for every weight within 2^-17 of
// the matrix maximum; the epilogues undo s exactly (fmaf(acc, 1/s, bias)).
//
// Every operand lives in HBM already in the shared-memory image of its tile ("tiled operand": for a tile of 128
// rows x 32 k, element (r, k) sits at  (k/8)*1024 + r*8 + k%8  — the K-major no-swizzle canonical layout of wgmma with
// core matrices of 8 rows x 16 B, SBO = 128 B between 8-row groups, LBO = 2048 B between the 8-element K chunks;
// weight tiles have 256 rows, LBO = 4096 B).  One producer thread moves whole tiles with cp.async.bulk (TMA engine, no
// tensor map) onto an mbarrier ring; two consumer warpgroups (64 rows each) issue wgmma.mma_async m64n256k16 straight
// from the ring, keep the 64 x 256 fp32 accumulator in registers (128 per thread), apply bias + cell in registers, and
// write the NEXT operand (h_t as hi/lo tiles), so activations never exist in fp32 in HBM between layers.
#pragma once
#include "common.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <type_traits>

namespace pb {
namespace tc {

// 16-bit operand type of the hi / lo split: fp16 (11 + 11 significant bits: a*w ~= a_hi*w_hi + a_hi*w_lo + a_lo*w_hi is
// good to ~2^-22 relative, 10-50 x closer to the fp32 reference than the bf16 split at the same three products per k-tile —
// scripts/sim_precision.py, DESIGN.md).  Activations are clamped to +-65504 (recurrent states are in [-1, 1]; MLP
// activations of O(1..10)); -DPB_OPERAND_BF16 selects the bf16 split (8 + 8 bits, no range limit).
#ifdef PB_OPERAND_BF16
typedef __nv_bfloat16 op_t;
#define OP_PTX "bf16"
__host__ __device__ __forceinline__ uint16_t op_bits(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }
__host__ __device__ __forceinline__ float op_val(uint32_t b) { return __bfloat162float(__ushort_as_bfloat16((unsigned short) (b & 0xffffu))); }
__device__ __forceinline__ uint16_t op_bits_unit(float v) { return op_bits(v); }
#else
typedef __half op_t;
#define OP_PTX "f16"
__host__ __device__ __forceinline__ uint16_t op_bits(float v) { return __half_as_ushort(__float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f))); }
__host__ __device__ __forceinline__ float op_val(uint32_t b) { return __half2float(__ushort_as_half((unsigned short) (b & 0xffffu))); }
// op_bits of a value with |v| <= 1 (LSTM hidden states), where the clamp is the identity
__device__ __forceinline__ uint16_t op_bits_unit(float v) { return __half_as_ushort(__float2half_rn(v)); }
#endif

constexpr int BM = 128, BK = 32;
constexpr int TILE_ELEMS = 128 * BK;                 // 4096 operand elements
constexpr int TILE_BYTES = TILE_ELEMS * 2;           // 8192
constexpr int PBN = 256;                             // output columns per tile = N of one wgmma
constexpr int PSTAGES = 4;
constexpr int WTILE_ELEMS = PBN * BK;                // weight tile image [kc][256 rows][8]
constexpr int WTILE_BYTES = WTILE_ELEMS * 2;
constexpr int PSTAGE_BYTES = 2 * TILE_BYTES + 2 * WTILE_BYTES;   // A_hi, A_lo, B_hi, B_lo = 48 KB
constexpr int PSMEM_BYTES = PSTAGES * PSTAGE_BYTES + 256;         // 192 KB ring + barriers: one CTA per SM
constexpr int CONS_WARPS = 8;                        // warps 0-7: two consumer warpgroups (rows 0-63, 64-127)
constexpr int PG_THREADS = 32 * CONS_WARPS + 32;     // + warp 8: producer
// k_lstm_layer: warps 8-11 form a producer warpgroup, so that setmaxnreg can move its registers to the consumers (one
// thread issues the copies); the direction's 1,024 bias floats sit behind the ring and the barriers
constexpr int LSTM_THREADS = 32 * CONS_WARPS + 128;
constexpr int LSTM_SMEM_BYTES = PSMEM_BYTES + 1024 * 4;
constexpr int LSTM_PROD_REGS = 40, LSTM_CONS_REGS = 232;   // 128 x 40 + 256 x 232 = 384 x 168, the launch's register file

enum { EPI_BIAS = 0, EPI_SELU = 1, EPI_LSTM = 2 };

struct Seg {                       // one K-segment of the A operand
    const op_t *hi, *lo;           // lo == nullptr: exactly representable operand (int8 images), a_lo*w_hi product skipped
    int64_t mt_stride;             // elements between consecutive row tiles
    int nkt;                       // k-tiles in this segment
};
struct Dir {
    Seg seg[2];
    const op_t *w_hi, *w_lo;            // [n_tile][w_nkt][WTILE_ELEMS]
    int w_nkt;                          // k-tiles per n-tile of the packed weight (>= k-tiles of this launch)
    const float *bias;                  // [N]
    float inv_scale;                    // 1 / s of the packed weight (TcRnn / TcLin::scale): acc * inv_scale + bias, exact
    float *c;                           // LSTM cell state of 256 units, lane-owned (c_index)
    op_t *y_hi, *y_lo;                  // output operand tiles: tile (mt, y_kt0 + col/32)
    int64_t y_mt_stride;
    int y_kt0;
    float *y_f32; int64_t ldy;          // optional fp32 copy  y_f32[row*ldy + col]
};
struct Args {
    Dir d[2];
    int M, N;                           // valid rows; N = columns of the packed weight (multiple of 256)
};

// Cell state of one direction of a 256-unit LSTM layer: 128 rows x 256 units = 32,768 floats per row tile, laid out so that
// each consumer thread's cells are contiguous.  In every LSTM epilogue consumer thread ct = 32 warp + lane (0-255) owns row
// r = 16 warp + lane / 4 + 8 (lane & 1) of its tile and units u with u & 1 = (lane >> 1) & 1; cell (u, r) sits at
//   ((u / 8) * 256 + ct) * 4 + (u / 2) % 4
// so a lane's four cells u / 8 = const go out as one 16 B access, and a warp's as 512 contiguous bytes.  A lane owns the
// same cells at every step, and nothing outside the layer kernels reads them except the test hooks (through this function).
__host__ __device__ __forceinline__ int64_t c_index(int unit, int64_t row) {
    const int r = (int) (row & 127);
    const int ct = (r >> 4) * 32 + (r & 7) * 4 + (unit & 1) * 2 + ((r >> 3) & 1);
    return (row >> 7) * (BM * 256) + ((int64_t) (unit >> 3) * 256 + ct) * 4 + ((unit >> 1) & 3);
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t) __cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// wgmma shared-memory descriptor: K-major, no swizzle, SBO = 128 B (8-row group stride), LBO = K chunk stride
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo) {
    uint64_t d = 0;
    d |= (uint64_t) ((addr >> 4) & 0x3FFF);
    d |= (uint64_t) ((lbo >> 4) & 0x3FFF) << 16;
    d |= (uint64_t) ((128u >> 4) & 0x3FFF) << 32;
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// per-warpgroup register budget (every warp of the warpgroup executes it)
template <int N>
__device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// d[64 x 256] += A[64 x 16] B[256 x 16]^T, both operands K-major in shared memory (descriptors), fp32 accumulate
__device__ __forceinline__ void wgmma_256(float (&d)[128], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32." OP_PTX "." OP_PTX " "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(adesc), "l"(bdesc), "r"(1));
}
// d[64 x 128] += A[64 x 16] B[128 x 16]^T (k_lstm_layer_enc's half gate tiles); each output gets the sums of wgmma_256
__device__ __forceinline__ void wgmma_128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." OP_PTX "." OP_PTX " "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(1));
}

// ---------------------------------------------------------------- int8-slice operands (mode 2: decoder LSTM layer and linear_1)
// A value v in [-1, 1] (an LSTM hidden state) is held as the 16-bit fixed-point integer q = rint(v * 32512) split into two
// signed int8 slices, q = 256 q1 + q0 with q1 = floor((q + 128) / 256) in [-127, 127] and q0 in [-128, 127].  A weight row
// (gate column n, K = [W_ih | W_hh]) is held the same way at its own scale sw_n = 32512 / max_k |W[n][k]|.  Three s8 x s8
// products with exact int32 accumulation, a1 w1 into acc_hh and a1 w0 + a0 w1 into acc_mix, give
//   A W^T ~= (65536 acc_hh + 256 acc_mix) / (32512 sw_n)
// dropping a0 w0 (<= 2^-16 of the product's range).  |acc_hh| <= 768 * 127^2 < 2^24 converts to fp32 exactly.
// Tiled slice operand ("QSeq"): per (row tile, time step) 8 k-tiles of 128 rows x 64 k, one byte per element at
// (k / 16) * 2048 + r * 16 + k % 16 (K-major no-swizzle canonical layout of 8-bit wgmma: core matrices 8 rows x 16 B, SBO
// 128 B, LBO 2048 B); feature f of direction d is k = d * 256 + f.  Weight k-tiles have the same layout with 128 gate
// columns for the 128 rows.
constexpr int QK = 64;                              // k per ring stage
constexpr int QTILE_BYTES = 128 * QK;               // 8 KB: one slice of a 128 x 64 tile
constexpr int QN = 128;                             // gate columns per tile (32 hidden units x 4 gates)
constexpr int QSTAGES = 6;                          // k_gemm_q8's ring
constexpr int QSTAGE_BYTES = 4 * QTILE_BYTES;       // a1, a0, w1, w0 = 32 KB
constexpr int GQSMEM_BYTES = QSTAGES * QSTAGE_BYTES + 256;                  // k_gemm_q8: ring + barriers
// k_lstm_layer_q8: a 4-stage ring, one gate tile's fp32 pre-activations (128 rows x 128 columns) staged for the epilogue
// warpgroup, barriers, bias and column scales = 205,056 B
constexpr int LQSTAGES = 4;
constexpr int QPRE_BYTES = BM * QN * 4;
constexpr int QSMEM_BYTES = LQSTAGES * QSTAGE_BYTES + QPRE_BYTES + 256 + 2 * 1024 * 4;
// warps 0-7 consumers, 8-11 the epilogue warpgroup, 12-15 the producer warpgroup (one issuing thread); the setmaxnreg split
// 24 + 2 x 168 + 152 = 4 x 128 is the launch's register file
constexpr int LQ_THREADS = 512;
constexpr int LQ_EPI_WARP = 8, LQ_PROD_WARP = 12;
constexpr int LQ_PROD_REGS = 24, LQ_CONS_REGS = 168, LQ_EPI_REGS = 152;
constexpr float QSCALE = 32512.f;

// d[64 x 128] (s32) += A[64 x 32] B[128 x 32]^T, s8 operands K-major in shared memory
__device__ __forceinline__ void wgmma_q8(int (&d)[64], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(1));
}
// u = q + 128 of a hidden value (the cell's h = sigm * tanh never leaves [-1, 1], so the clamp is the identity).  The slice
// q1 = u >> 8 is byte 1 of u, and the byte of q0 = q - 256 q1 is byte 0 of u with its top bit flipped.
__device__ __forceinline__ int qbias(float v) { return __float2int_rn(v * QSCALE) + 128; }
// one slice (lo: q0, else q1) of four consecutive units, one byte each, from their qbias values
__device__ __forceinline__ uint32_t qword(int u0, int u1, int u2, int u3, bool lo) {
    const uint32_t sel = lo ? 0x40u : 0x51u;
    const uint32_t w = __byte_perm(__byte_perm(u0, u1, sel), __byte_perm(u2, u3, sel), 0x5410);
    return lo ? w ^ 0x80808080u : w;
}

// exp via ex2.approx (2 ulp) + fast divide: absolute error ~1e-6, far inside the 1e-3 parity tolerance.  exp_ftz is __expf
// without its fix-up for results below 2^-126 (flushed to zero instead): the bits differ only where 1 + e rounds to 1
// either way (sigm), and never occur in tanh_fast (e >= e^-30).
__device__ __forceinline__ float exp_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
    return y;
}
__device__ __forceinline__ float sigm(float x) { return __fdividef(1.0f, 1.0f + exp_ftz(-x)); }
__device__ __forceinline__ float tanh_fast(float x) {
    const float e = exp_ftz(2.0f * fminf(fmaxf(x, -15.0f), 15.0f));
    return 1.0f - __fdividef(2.0f, e + 1.0f);
}
__device__ __forceinline__ float selu(float x) {
    const float alpha = 1.6732632423543772848170429916717f, scale = 1.0507009873554804934193349852946f;
    return x > 0.f ? scale * x : scale * alpha * (__expf(x) - 1.0f);
}
// 2 fp32 -> 2 hi + 2 lo 16-bit operands, 4 B each.  UNIT: |a|, |b| <= 1, no range clamp needed (same bits)
template <bool UNIT = false>
__device__ __forceinline__ void split2(float a, float b, uint32_t &hi, uint32_t &lo) {
    const uint16_t h0 = UNIT ? op_bits_unit(a) : op_bits(a), h1 = UNIT ? op_bits_unit(b) : op_bits(b);
    const uint16_t l0 = UNIT ? op_bits_unit(a - op_val(h0)) : op_bits(a - op_val(h0));
    const uint16_t l1 = UNIT ? op_bits_unit(b - op_val(h1)) : op_bits(b - op_val(h1));
    hi = (uint32_t) h0 | ((uint32_t) h1 << 16);
    lo = (uint32_t) l0 | ((uint32_t) l1 << 16);
}
// element (r, k) of a tiled operand, relative to its tile
__device__ __forceinline__ int64_t tile_off(int k, int r128) { return (int64_t) (k >> 5) * TILE_ELEMS + ((k & 31) >> 3) * 1024 + r128 * 8 + (k & 7); }

// Producer: one k-tile (A hi [+ lo], B hi + lo) into ring stage `g % PSTAGES` once the consumers have released it.
__device__ __forceinline__ void load_stage(uint32_t smem_base, uint32_t bar_full, uint32_t bar_empty, uint32_t g, const op_t *a_hi,
                                           const op_t *a_lo, const op_t *w_hi, const op_t *w_lo) {
    const uint32_t s = g % PSTAGES, ph = (g / PSTAGES) & 1u;
    mbar_wait(bar_empty + 8 * s, ph ^ 1u);
    const uint32_t st = smem_base + s * PSTAGE_BYTES;
    mbar_expect_tx(bar_full + 8 * s, (a_lo ? 2u : 1u) * TILE_BYTES + 2u * WTILE_BYTES);
    bulk_g2s(st, a_hi, TILE_BYTES, bar_full + 8 * s);
    if (a_lo) bulk_g2s(st + TILE_BYTES, a_lo, TILE_BYTES, bar_full + 8 * s);
    bulk_g2s(st + 2 * TILE_BYTES, w_hi, WTILE_BYTES, bar_full + 8 * s);
    bulk_g2s(st + 2 * TILE_BYTES + WTILE_BYTES, w_lo, WTILE_BYTES, bar_full + 8 * s);
}

// The products of one k-tile as one committed wgmma group; LO adds a_lo x w_hi.  Both variants are complete groups, so the
// choice between them is a branch around whole groups (a lone conditional wgmma makes ptxas serialize every wgmma).
template <bool LO>
__device__ __forceinline__ void mma_ktile(float (&acc)[128], uint32_t st, uint32_t a) {
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < BK / 16; ks++) {
        const uint64_t a_hi = smem_desc(a + ks * 4096, 2048);
        const uint64_t b_hi = smem_desc(st + 2 * TILE_BYTES + ks * 8192, 4096);
        const uint64_t b_lo = smem_desc(st + 2 * TILE_BYTES + WTILE_BYTES + ks * 8192, 4096);
        wgmma_256(acc, a_hi, b_hi);
        wgmma_256(acc, a_hi, b_lo);
        if (LO) wgmma_256(acc, smem_desc(a + TILE_BYTES + ks * 4096, 2048), b_hi);
    }
    wg_commit();
}

// Consumer warpgroup `wg`: acc (rows 64 wg .. 64 wg + 63 of the tile) = sum over `nkt` ring k-tiles.  k-tiles below
// `nkt0` run the a_lo x w_hi product when lo0, the others when lo1.  Each stage is released as soon as the wgmma group
// that read it has completed, so the producer refills it while the next k-tile multiplies.
__device__ __forceinline__ void mma_tile(float (&acc)[128], uint32_t smem_base, uint32_t bar_full, uint32_t bar_empty, uint32_t &g,
                                         int nkt, int nkt0, bool lo0, bool lo1, int wg, int lane) {
#pragma unroll
    for (int i = 0; i < 128; i++) acc[i] = 0.f;
    for (int kt = 0; kt < nkt; kt++, g++) {
        const uint32_t s = g % PSTAGES, ph = (g / PSTAGES) & 1u;
        mbar_wait(bar_full + 8 * s, ph);
        const bool lo = kt < nkt0 ? lo0 : lo1;
        const uint32_t st = smem_base + s * PSTAGE_BYTES, a = st + (uint32_t) wg * 1024;
        if (lo) mma_ktile<true>(acc, st, a);
        else mma_ktile<false>(acc, st, a);
        wg_wait<1>();
        if (kt > 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8 * ((g - 1) % PSTAGES));
        }
    }
    wg_wait<0>();
    if (nkt > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * ((g - 1) % PSTAGES));
    }
}

// Accumulator fragment of m64n256: acc[4i + e] is row rA + 8 * (e >> 1), column 8i + 2q + (e & 1), with
// rA = 16 * (warp % 4) + lane / 4 (+ 64 for the second warpgroup) and q = lane % 4.  Gate columns are interleaved per
// hidden unit (column 4u + gate), so lane pairs (q, q ^ 1) hold gates {0, 1} and {2, 3} of units 2i + q / 2 for both rows:
// one exchange gives the even lane all four gates of row rA and the odd lane those of row rA + 8.
// The packed weights carry a power-of-two scale s, undone exactly by the multiply of the fused multiply-add with the bias.
// The m64n128 fragment (NACC = 64) is the first half of this one: i < 16, columns of its own 128-column tile.
template <int NACC>
__device__ __forceinline__ void gates4(const float (&acc)[NACC], int i, float2 bz, float inv_s, int q, float (&gt)[4]) {
    const float a0 = fmaf(acc[4 * i + 0], inv_s, bz.x), a1 = fmaf(acc[4 * i + 1], inv_s, bz.y);
    const float b0 = fmaf(acc[4 * i + 2], inv_s, bz.x), b1 = fmaf(acc[4 * i + 3], inv_s, bz.y);
    const bool odd = q & 1;
    const float r0 = __shfl_xor_sync(0xffffffffu, odd ? a0 : b0, 1);
    const float r1 = __shfl_xor_sync(0xffffffffu, odd ? a1 : b1, 1);
    gt[0] = odd ? r0 : a0; gt[1] = odd ? r1 : a1;
    gt[2] = odd ? b0 : r0; gt[3] = odd ? b1 : r1;
}
// h of units (2i, 2i + 1) meet in lanes q and q ^ 2: the even-unit lane stores both (4 B operand words, 8 B fp32 pair)
__device__ __forceinline__ void store_h(float hn, bool store, op_t *y_hi, op_t *y_lo, int64_t o, float *y_f32) {
    uint32_t hi, lo;
    const float hn1 = __shfl_xor_sync(0xffffffffu, hn, 2);
    split2(hn, hn1, hi, lo);
    // predicated stores, no branch: a branch per cell would keep the scheduler from overlapping consecutive cells
    if (store) *reinterpret_cast<uint32_t *>(y_hi + o) = hi;
    if (store) *reinterpret_cast<uint32_t *>(y_lo + o) = lo;
    if (store && y_f32) *reinterpret_cast<float2 *>(y_f32) = make_float2(hn, hn1);
}
__device__ __forceinline__ float load_h(const op_t *hi, const op_t *lo, int64_t o) {
    return op_val(reinterpret_cast<const uint16_t *>(hi)[o]) + op_val(reinterpret_cast<const uint16_t *>(lo)[o]);
}

// ---------------------------------------------------------------- persistent GEMM
// One CTA per SM loops over 128 x 256 output tiles (static round-robin); the producer runs ahead across tiles, so the
// next tile's operands stream in while the consumers apply the epilogue of the current one.
template <int EPI>
__global__ void __launch_bounds__(PG_THREADS, 1) k_tc_gemm_p(Args G, int n_mt, int n_nt /* 256-column tiles */, int n_dir) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + PSTAGES * PSTAGE_BYTES);
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + PSTAGES);
    const uint32_t smem_base = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tiles = n_mt * n_nt * n_dir;

    if (threadIdx.x == 0) {
        for (int s = 0; s < PSTAGES; s++) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, CONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // tile -> (dir, mt, nt): nt fastest so that CTAs running together share the A row tile
    auto decode = [&](int tile, int &dir, int &mt, int &nt) {
        nt = tile % n_nt;
        const int r = tile / n_nt;
        mt = r % n_mt;
        dir = r / n_mt;
    };

    if (warp == CONS_WARPS) {
        if (lane == 0) {
            uint32_t g = 0;                                   // running k-tile counter across tiles
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                int dir, mt, nt;
                decode(tile, dir, mt, nt);
                const Dir &D = G.d[dir];
                const int nkt0 = D.seg[0].nkt, nkt = nkt0 + D.seg[1].nkt;
                for (int kt = 0; kt < nkt; kt++, g++) {
                    const Seg &S = (kt < nkt0) ? D.seg[0] : D.seg[1];
                    const int64_t off = (int64_t) mt * S.mt_stride + (int64_t) ((kt < nkt0) ? kt : kt - nkt0) * TILE_ELEMS;
                    const int64_t woff = ((int64_t) nt * D.w_nkt + kt) * WTILE_ELEMS;
                    load_stage(smem_base, bar_full, bar_empty, g, S.hi + off, S.lo ? S.lo + off : nullptr, D.w_hi + woff, D.w_lo + woff);
                }
            }
        }
        return;
    }
    const int wg = warp >> 2, q = lane & 3;
    const int rA = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    uint32_t g = 0;
    float acc[128];
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int dir, mt, nt;
        decode(tile, dir, mt, nt);
        const Dir &D = G.d[dir];
        mma_tile(acc, smem_base, bar_full, bar_empty, g, D.seg[0].nkt + D.seg[1].nkt, D.seg[0].nkt, D.seg[0].lo != nullptr,
                 D.seg[1].lo != nullptr, wg, lane);
        if (EPI == EPI_BIAS || EPI == EPI_SELU) {
#pragma unroll
            for (int i = 0; i < PBN / 8; i++) {
                const int col = nt * PBN + 8 * i + 2 * q;
                const float2 bz = __ldg(reinterpret_cast<const float2 *>(D.bias + col));
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int r128 = rA + 8 * h, row = mt * BM + r128;
                    float v0 = fmaf(acc[4 * i + 2 * h], D.inv_scale, bz.x), v1 = fmaf(acc[4 * i + 2 * h + 1], D.inv_scale, bz.y);
                    if (EPI == EPI_SELU) { v0 = selu(v0); v1 = selu(v1); }
                    if (row < G.M) {
                        if (D.y_hi) {
                            uint32_t hi, lo;
                            split2(v0, v1, hi, lo);
                            const int64_t o = (int64_t) mt * D.y_mt_stride + (int64_t) D.y_kt0 * TILE_ELEMS + tile_off(col, r128);
                            *reinterpret_cast<uint32_t *>(D.y_hi + o) = hi;
                            *reinterpret_cast<uint32_t *>(D.y_lo + o) = lo;
                        }
                        if (D.y_f32) *reinterpret_cast<float2 *>(D.y_f32 + (int64_t) row * D.ldy + col) = make_float2(v0, v1);
                    }
                }
            }
        } else {
            const int r128 = rA + 8 * (q & 1), row = mt * BM + r128;
            const bool valid = row < G.M;
            // unit nt * 64 + 2 i + q / 2 of this row sits at cl + (i / 4) * 1024 + i % 4 (c_index)
            float *const cl = D.c + c_index(nt * (PBN / 4) + (q >> 1), row);
#pragma unroll
            for (int i = 0; i < PBN / 8; i++) {
                const int j = nt * (PBN / 4) + 2 * i + (q >> 1);
                float gt[4];
                gates4(acc, i, __ldg(reinterpret_cast<const float2 *>(D.bias + nt * PBN + 8 * i + 2 * q)), D.inv_scale, q, gt);
                float *cp = cl + (i >> 2) * 1024 + (i & 3);
                const float cn = sigm(gt[1]) * (valid ? *cp : 0.f) + sigm(gt[0]) * tanh_fast(gt[2]);
                if (valid) *cp = cn;
                const float hn = sigm(gt[3]) * tanh_fast(cn);
                const int64_t o = (int64_t) mt * D.y_mt_stride + (int64_t) D.y_kt0 * TILE_ELEMS + tile_off(j, r128);
                store_h(hn, valid && !(q & 2), D.y_hi, D.y_lo, o, D.y_f32 ? D.y_f32 + (int64_t) row * D.ldy + j : nullptr);
            }
        }
    }
}

// ---------------------------------------------------------------- persistent LSTM layer kernel (variant)
// All T time steps of one bidirectional LSTM layer in ONE launch.  CTA b owns (direction, 128-candidate row tile) for the
// whole sequence and computes all four 256-column gate tiles of every step itself, so the recurrence never leaves the
// CTA: the consumers write h_t as hi/lo operand tiles into the layer's output sequence, arrive on a CTA-local mbarrier,
// and the producer thread loads those tiles back as the h-part of step t+1 (generic -> async proxy fence in between).
// The x-part of step t+1 (1 k-tile for the encoder layer, 16 for the decoder layer) does not depend on h_t and is
// streamed while the last epilogue of step t runs.  One chunk of 8,448 candidates = 66 row tiles x 2 directions = 132
// CTAs = one per H100 SM; the per-step kernel above stays as the cross-check path.
// Both consumer warpgroups (64 rows each) multiply a 256-column gate tile together, then both run its epilogue.
// The epilogue touches no global load: each consumer lane loads the 32 cell states of its (row, unit) cells of a gate tile
// before that tile's k-loop, so they arrive under the MMA (a lane owns the same cells at every step: its own store of step
// t-1 precedes the load in program order), and the bias is staged in shared memory once per launch.
struct LstmLayer {
    const op_t *x_hi, *x_lo;           // input sequence operand: tile (mt, t, kt) at mt * x_mt_stride + (t * x_nkt + kt) * TILE_ELEMS
    int64_t x_mt_stride;
    int x_nkt;
    const op_t *w_hi[2], *w_lo[2];     // per direction: [4 n-tiles][x_nkt + 8][WTILE_ELEMS]
    const float *bias[2];
    float inv_scale[2];                // 1 / s of each direction's packed weight
    float *c[2];                       // cell state per direction (c_index), zero initialised
    op_t *y_hi, *y_lo;                 // output sequence operand [mt][T][16] tiles; (time tt, direction d) -> k-tiles tt * 16 + d * 8 ...
    int64_t y_mt_stride;
    float *y_f32;                      // optional fp32 copy [row][T][512]
    int64_t ldy;
    int M, n_mt, T;
    int lo_x, lo_h;                    // 1: the a_lo x w_hi product of the x-part / h-part is executed (0: two products)
    int8_t *q1, *q0;                   // k_lstm_layer_enc: h_t as int8 slices for the next layer instead of y_lo (QSeq layout)
    int64_t q_mt_stride;               // bytes
    const op_t *wh_hi[2], *wh_lo[2];   // k_lstm_layer_enc, per direction: [8 half tiles][x_nkt + 8][TILE_ELEMS] (128 gate columns)
#ifdef PB_LSTM_TRACE
    uint64_t *trace;                   // lstm_trace_words(T) stamps per launch, nullptr: none
#endif
};

#ifdef PB_LSTM_TRACE
// Timing build only (-DPB_LSTM_TRACE; scripts/trace_lstm_layer.py): %clock64 stamps of CTAs 0, gridDim / 2 and
// gridDim - 1 of k_lstm_layer and k_lstm_layer_q8.  Per sampled CTA, in 64-bit words (cw = consumer warp 0-7, nt = gate
// tile: 0-3 in k_lstm_layer, 0-7 in k_lstm_layer_q8):
//   [((cw * T + t) * 8 + nt) * 4 + k]  k: 0 tile start, 1 first bar_full passed, 2 wg_wait<0> returned, 3 epilogue end
//   [256 T + (cw * T + t) * 2 + k]     k: 0 __threadfence returned, 1 bar_h arrived
//   [272 T + t * 3 + k]                producer, t >= 1; k: 0 bar_h wait start, 1 wait end, 2 first h-part copy issued
//   [275 T + k]                        k: 0 %globaltimer, 1 %clock64 at the start; 2, 3 the same when warp 0 ends
//   [275 T + 4 + ((ew * T + t) * 8 + nt) * 4 + k]   k_lstm_layer_q8's epilogue warps ew = 0-3; k: 0 "staged" wait issued,
//                                      1 cells done (slices and c stored), 2 h_t published (bar_h arrived; nt = 7 only).
//                                      bar.sync defers its blocking to the next memory access, so a clock read right after
//                                      it would not mark the release: the consumers' "staging stored" stamps bound it.
// k_lstm_layer_enc (no bar_h, producer words stay 0): nt = half tile 0-7 with k: 0 start, 1 first bar_full passed, 2 last
// k-tile issued, 3 end (the previous half's epilogue runs between 1 and 2); the step words are 0 half 7's epilogue done,
// 1 h published (named barrier passed), both inside half 0 of step t.  In k_lstm_layer_q8 the consumers' k = 3 is
// "staging stored" and their step words stay 0 (the epilogue warps publish h).
constexpr int LSTM_TRACE_CTAS = 3;
__host__ __device__ constexpr int64_t lstm_trace_cta_words(int T) { return 403 * (int64_t) T + 4; }
__host__ __device__ constexpr int64_t lstm_trace_words(int T) { return LSTM_TRACE_CTAS * lstm_trace_cta_words(T); }
__device__ __forceinline__ uint64_t trace_clock() {
    uint64_t c;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(c) :: "memory");
    return c;
}
__device__ __forceinline__ uint64_t trace_gtime() {
    uint64_t c;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(c) :: "memory");
    return c;
}
#define LSTM_STAMP(off)                                          \
    do {                                                         \
        if (tr && lane == 0) tr[off] = trace_clock();            \
    } while (0)
#else
#define LSTM_STAMP(off) do {} while (0)
#endif

__global__ void __launch_bounds__(LSTM_THREADS, 1) k_lstm_layer(LstmLayer G) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + PSTAGES * PSTAGE_BYTES);
    float *sbias = reinterpret_cast<float *>(smem + PSMEM_BYTES);
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + PSTAGES), bar_h = smem_u32(bars + 2 * PSTAGES);
    const uint32_t smem_base = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.x / G.n_mt, mt = blockIdx.x % G.n_mt;
    const int w_nkt = G.x_nkt + 8;

    if (threadIdx.x == 0) {
        for (int s = 0; s < PSTAGES; s++) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, CONS_WARPS); }
        mbar_init(bar_h, CONS_WARPS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < 4 * PBN; i += LSTM_THREADS) sbias[i] = G.bias[dir][i];
#ifdef PB_LSTM_TRACE
    const int ts = blockIdx.x == 0 ? 0 : blockIdx.x == gridDim.x / 2 ? 1 : blockIdx.x == gridDim.x - 1 ? 2 : -1;
    uint64_t *const tr = G.trace && ts >= 0 ? G.trace + ts * lstm_trace_cta_words(G.T) : nullptr;
    if (tr && threadIdx.x == 0) { tr[275 * G.T] = trace_gtime(); tr[275 * G.T + 1] = trace_clock(); }
#endif
    __syncthreads();

    if (warp >= CONS_WARPS) {
        reg_dealloc<LSTM_PROD_REGS>();
        if (threadIdx.x == 32 * CONS_WARPS) {
            uint32_t g = 0;
            for (int t = 0; t < G.T; t++) {
                const int tt = dir ? G.T - 1 - t : t, tp = dir ? tt + 1 : tt - 1;
                const int nkt = G.x_nkt + (t > 0 ? 8 : 0);
                for (int nt = 0; nt < 4; nt++) {
                    for (int kt = 0; kt < nkt; kt++, g++) {
                        const op_t *a_hi, *a_lo;
                        if (kt < G.x_nkt) {
                            const int64_t off = (int64_t) mt * G.x_mt_stride + ((int64_t) tt * G.x_nkt + kt) * TILE_ELEMS;
                            a_hi = G.x_hi + off; a_lo = (G.x_lo && G.lo_x) ? G.x_lo + off : nullptr;
                        } else {
                            const int kk = kt - G.x_nkt;
                            if (kk == 0 && nt == 0) {
                                // every consumer warp has written its part of h_{t-1}: make it visible to the bulk-copy engine
                                LSTM_STAMP(272 * G.T + t * 3);
                                mbar_wait(bar_h, (uint32_t) (t - 1) & 1u);
                                asm volatile("fence.proxy.async;" ::: "memory");
                                LSTM_STAMP(272 * G.T + t * 3 + 1);
                            }
                            const int64_t off = (int64_t) mt * G.y_mt_stride + ((int64_t) tp * 16 + dir * 8 + kk) * TILE_ELEMS;
                            a_hi = G.y_hi + off; a_lo = G.lo_h ? G.y_lo + off : nullptr;
                        }
                        const int64_t woff = ((int64_t) nt * w_nkt + kt) * WTILE_ELEMS;
                        load_stage(smem_base, bar_full, bar_empty, g, a_hi, a_lo, G.w_hi[dir] + woff, G.w_lo[dir] + woff);
                        if (t > 0 && nt == 0 && kt == G.x_nkt) LSTM_STAMP(272 * G.T + t * 3 + 2);
                    }
                }
            }
        }
        return;
    }
    reg_alloc<LSTM_CONS_REGS>();
    const int wg = warp >> 2, q = lane & 3;
    const int r128 = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * (q & 1);      // row of this lane's cells
    const int row = mt * BM + r128;
    const bool valid = row < G.M;
    const bool lo_x = G.x_lo != nullptr && G.lo_x != 0, lo_h = G.lo_h != 0;
    const float inv_s = G.inv_scale[dir];
    float4 *const cl = reinterpret_cast<float4 *>(G.c[dir] + c_index(q >> 1, row));   // this lane's first four cells
    uint32_t g = 0;
    float acc[128];
    for (int t = 0; t < G.T; t++) {
        const int tt = dir ? G.T - 1 - t : t;
        const int nkt = G.x_nkt + (t > 0 ? 8 : 0);
        const int64_t y0 = (int64_t) mt * G.y_mt_stride + (int64_t) (tt * 16 + dir * 8) * TILE_ELEMS + r128 * 8;
        for (int nt = 0; nt < 4; nt++) {
#ifdef PB_LSTM_TRACE
            const int tc0 = ((warp * G.T + t) * 8 + nt) * 4;
#endif
            LSTM_STAMP(tc0);
            // cell states of units nt * 64 + 2 i + q / 2 (cells 4 k .. 4 k + 3 in one float4), in flight during the k-loop
            float4 *cp = cl + nt * (PBN / 32) * 256;
            float c_prev[PBN / 8];
#pragma unroll
            for (int k = 0; k < PBN / 32; k++) {
                const float4 v = valid ? __ldcg(cp + k * 256) : make_float4(0.f, 0.f, 0.f, 0.f);
                c_prev[4 * k] = v.x; c_prev[4 * k + 1] = v.y; c_prev[4 * k + 2] = v.z; c_prev[4 * k + 3] = v.w;
            }
#ifdef PB_LSTM_TRACE
            mbar_wait(bar_full + 8 * (g % PSTAGES), (g / PSTAGES) & 1u);     // mma_tile's first wait then passes at once
            LSTM_STAMP(tc0 + 1);
#endif
            mma_tile(acc, smem_base, bar_full, bar_empty, g, nkt, G.x_nkt, lo_x, lo_h, wg, lane);
            LSTM_STAMP(tc0 + 2);
            const float *sb = sbias + nt * PBN + 2 * q;
            // units nt * 64 .. + 63 are operand k-tiles 2 nt, 2 nt + 1 of this step.  Lanes q and q ^ 2 hold units 2 i and
            // 2 i + 1 of the same row: the even-unit lane writes the hi words of the pair, the odd-unit lane the lo words.
            const bool odd_u = q >> 1;
            op_t *yw = (odd_u ? G.y_lo : G.y_hi) + y0 + 2 * nt * TILE_ELEMS;
            float *yf = G.y_f32 ? G.y_f32 + (int64_t) row * G.ldy + (int64_t) tt * 512 + dir * 256 + nt * (PBN / 4) : nullptr;
#pragma unroll
            for (int m = 0; m < PBN / 16; m++) {
                // cells i = 2 m, 2 m + 1: their two 4 B operand words are adjacent in row r128 and go out as one 8 B store
                // (lanes 4 apart fill the other half of the 32 B sector); four cells per 16 B store need registers the
                // 168-register launch does not have (68 B of spills)
                uint32_t w[2];
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int i = 2 * m + e;
                    float gt[4];
                    gates4(acc, i, *reinterpret_cast<const float2 *>(sb + 8 * i), inv_s, q, gt);
                    const float cn = sigm(gt[1]) * c_prev[i] + sigm(gt[0]) * tanh_fast(gt[2]);
                    const float hn = sigm(gt[3]) * tanh_fast(cn);
                    c_prev[i] = cn;
                    const float hp = __shfl_xor_sync(0xffffffffu, hn, 2);
                    const float h0 = odd_u ? hp : hn, h1 = odd_u ? hn : hp;          // units 2 i, 2 i + 1
                    uint32_t hi, lo;
                    split2<true>(h0, h1, hi, lo);
                    w[e] = odd_u ? lo : hi;
                    if (yf && valid && !odd_u) *reinterpret_cast<float2 *>(yf + 2 * i) = make_float2(h0, h1);
                }
                // element (unit nt * 64 + 4 m, row r128) of the step's operand tiles, relative to the lane's base
                if (valid) __stwb(reinterpret_cast<uint2 *>(yw + (m >> 3) * TILE_ELEMS + ((m >> 1) & 3) * 1024 + 4 * (m & 1)), make_uint2(w[0], w[1]));
                // cells 2 m - 2 .. 2 m + 1 are done: one 16 B store
                if ((m & 1) && valid) {
                    const int k = m >> 1;
                    cp[k * 256] = make_float4(c_prev[4 * k], c_prev[4 * k + 1], c_prev[4 * k + 2], c_prev[4 * k + 3]);
                }
            }
            LSTM_STAMP(tc0 + 3);
        }
        // h_t of this warp's rows is complete (all four gate tiles): publish it to the producer thread
        __threadfence();
        LSTM_STAMP(256 * G.T + (warp * G.T + t) * 2);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_h);
        LSTM_STAMP(256 * G.T + (warp * G.T + t) * 2 + 1);
    }
#ifdef PB_LSTM_TRACE
    if (tr && threadIdx.x == 0) { tr[275 * G.T + 2] = trace_gtime(); tr[275 * G.T + 3] = trace_clock(); }
#endif
}

// ---------------------------------------------------------------- persistent encoder LSTM layer, h on chip (variant)
// k_lstm_layer's grid and arithmetic for the encoder layer with a hi-only h-part (lo_h == 0, x = the int8 images, 1 k-tile).
// Two changes:
//  * h stays in shared memory.  A warpgroup's h-part at step t + 1 is exactly the rows its own epilogues wrote at step t, so
//    each epilogue also writes its hi words into the step's shared h-part (operand tile layout, double-buffered by step
//    parity), and a per-warpgroup named barrier after a generic -> async proxy fence replaces bar_h, the __threadfence and
//    the producer's reload of h through L2.  The global h stores are k_lstm_layer's (y_hi and the odd lanes' y_lo words,
//    y_f32), except that Q8 writes the decoder's int8 slices alone (enc_cells); the next layer and the test hooks read them,
//    nothing in this kernel does.
//  * Each step is 8 half gate tiles of 128 columns (32 units x 4 gates, m64n128) into two accumulator sets, and the cell
//    epilogue of half h runs one unit pair per k-tile between the wgmma groups of half h + 1, so the tensor cores stay busy
//    while it runs.  Each output element gets the same products in the same order as in k_lstm_layer.
// The ring carries the 16 KB of weights (hi + lo) of one half-tile k-tile, from the half-tile packing wh_hi / wh_lo; the step's
// image k-tile has a two-slot buffer of its own, loaded once per step.  Shared memory: 2 x 64 KB h + 2 x 8 KB x + 4 x 16 KB
// ring + 4 KB bias + barriers = 217,344 B.
// At a step boundary the x k-tile and the h k-tiles 0-6 of half 0 (written by halves 0-6, published by the barrier after
// half 6's epilogue) run under half 7's epilogue; only h k-tile 7 waits for it.
constexpr int EH_BYTES = 8 * TILE_BYTES;                         // one step's h-part: 8 k-tiles of 128 rows
constexpr int ESTAGES = 4;
constexpr int ESTAGE_BYTES = 2 * TILE_BYTES;                     // W hi + lo of one half-tile k-tile
constexpr int ENC_NKT = 9;                                       // k-tiles per half tile from step 1 on: [x | h 0..7]
constexpr int ESMEM_BYTES = 2 * EH_BYTES + 2 * TILE_BYTES + ESTAGES * ESTAGE_BYTES + 1024 * 4 + 256;

// where the epilogue of one half tile writes: bias, cell states, global h words / slices / fp32 copy, shared h words
struct EncEpi {
    const float *sb;
    float4 *cp;
    op_t *yw;
    int8_t *qw;
    float *yf;
    uint32_t hs;
};

// Cells 2 m, 2 m + 1 of the lane's 16 in a half tile: k_lstm_layer's epilogue arithmetic and stores.  Q8: h_t leaves the
// kernel only as the decoder's two int8 slices (the even-unit lane writes q1, the odd-unit lane q0 of a unit pair): the fp16
// hi words' one reader was the layer's own h-part, now in shared memory, and the lo words have none (hi-only h-part).
template <bool Q8>
__device__ __forceinline__ void enc_cells(const float (&acc)[64], float (&c)[16], int m, const EncEpi &E, float inv_s, int q,
                                          bool odd_u, bool valid) {
    uint32_t w[2];
    int uq[4];
#pragma unroll
    for (int e = 0; e < 2; e++) {
        const int i = 2 * m + e;
        float gt[4];
        gates4(acc, i, *reinterpret_cast<const float2 *>(E.sb + 8 * i), inv_s, q, gt);
        const float cn = sigm(gt[1]) * c[i] + sigm(gt[0]) * tanh_fast(gt[2]);
        const float hn = sigm(gt[3]) * tanh_fast(cn);
        c[i] = cn;
        const float hp = __shfl_xor_sync(0xffffffffu, hn, 2);
        const float h0 = odd_u ? hp : hn, h1 = odd_u ? hn : hp;          // units 2 i, 2 i + 1
        if constexpr (Q8) {
            uq[2 * e] = qbias(h0); uq[2 * e + 1] = qbias(h1);
            w[e] = (uint32_t) op_bits_unit(h0) | ((uint32_t) op_bits_unit(h1) << 16);
        } else {
            uint32_t hi, lo;
            split2<true>(h0, h1, hi, lo);
            w[e] = odd_u ? lo : hi;
        }
        if (E.yf && valid && !odd_u) *reinterpret_cast<float2 *>(E.yf + 2 * i) = make_float2(h0, h1);
    }
    // element (unit 4 m of the half, row r128) of its operand k-tile, relative to the lane's base
    const int o = ((m >> 1) & 3) * 1024 + 4 * (m & 1);
    if constexpr (Q8) {
        if (valid) __stwb(reinterpret_cast<uint32_t *>(E.qw + (m >> 2) * 2048 + 4 * (m & 3)), qword(uq[0], uq[1], uq[2], uq[3], odd_u));
    } else {
        if (valid) __stwb(reinterpret_cast<uint2 *>(E.yw + o), make_uint2(w[0], w[1]));
    }
    // the next step's h-part: hi words of every row (a padding row's h only meets its own row of the product)
    if (!odd_u) asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(E.hs + 2 * o), "r"(w[0]), "r"(w[1]) : "memory");
    if ((m & 1) && valid) {
        const int k = m >> 1;
        E.cp[k * 256] = make_float4(c[4 * k], c[4 * k + 1], c[4 * k + 2], c[4 * k + 3]);
    }
}

// one k-tile of a half tile as one committed wgmma group: a_hi x w_hi + a_hi x w_lo per 16-k slice (mma_ktile<false>)
__device__ __forceinline__ void enc_ktile(float (&acc)[64], uint32_t a, uint32_t st) {
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < BK / 16; ks++) {
        const uint64_t a_hi = smem_desc(a + ks * 4096, 2048);
        wgmma_128(acc, a_hi, smem_desc(st + ks * 4096, 2048));
        wgmma_128(acc, a_hi, smem_desc(st + TILE_BYTES + ks * 4096, 2048));
    }
    wg_commit();
}

// this warpgroup's h words written so far are visible to its wgmma reads (all 4 warps' generic stores -> async proxy)
__device__ __forceinline__ void enc_publish_h(int wg) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
}

template <bool Q8>
__global__ void __launch_bounds__(LSTM_THREADS, 1) k_lstm_layer_enc(LstmLayer G) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int RING = 2 * EH_BYTES + 2 * TILE_BYTES, BIAS = RING + ESTAGES * ESTAGE_BYTES;
    float *sbias = reinterpret_cast<float *>(smem + BIAS);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + BIAS + 1024 * 4);
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + ESTAGES);
    const uint32_t bar_xfull = smem_u32(bars + 2 * ESTAGES), bar_xempty = smem_u32(bars + 2 * ESTAGES + 2);
    const uint32_t hbuf = smem_u32(smem), xbuf = hbuf + 2 * EH_BYTES, ring = hbuf + RING;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.x / G.n_mt, mt = blockIdx.x % G.n_mt;

    if (threadIdx.x == 0) {
        for (int s = 0; s < ESTAGES; s++) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, CONS_WARPS); }
        for (int s = 0; s < 2; s++) { mbar_init(bar_xfull + 8 * s, 1); mbar_init(bar_xempty + 8 * s, CONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < 4 * PBN; i += LSTM_THREADS) sbias[i] = G.bias[dir][i];
#ifdef PB_LSTM_TRACE
    const int ts = blockIdx.x == 0 ? 0 : blockIdx.x == gridDim.x / 2 ? 1 : blockIdx.x == gridDim.x - 1 ? 2 : -1;
    uint64_t *const tr = G.trace && ts >= 0 ? G.trace + ts * lstm_trace_cta_words(G.T) : nullptr;
    if (tr && threadIdx.x == 0) { tr[275 * G.T] = trace_gtime(); tr[275 * G.T + 1] = trace_clock(); }
#endif
    __syncthreads();

    if (warp >= CONS_WARPS) {
        reg_dealloc<LSTM_PROD_REGS>();
        if (threadIdx.x == 32 * CONS_WARPS) {
            uint32_t g = 0;
            for (int t = 0; t < G.T; t++) {
                const int tt = dir ? G.T - 1 - t : t;
                const uint32_t xs = (uint32_t) t & 1u;
                mbar_wait(bar_xempty + 8 * xs, (((uint32_t) t >> 1) & 1u) ^ 1u);
                mbar_expect_tx(bar_xfull + 8 * xs, TILE_BYTES);
                bulk_g2s(xbuf + xs * TILE_BYTES, G.x_hi + (int64_t) mt * G.x_mt_stride + (int64_t) tt * TILE_ELEMS, TILE_BYTES, bar_xfull + 8 * xs);
                const int nkt = t > 0 ? ENC_NKT : 1;
                for (int h = 0; h < 8; h++)
                    for (int kt = 0; kt < nkt; kt++, g++) {
                        const uint32_t s = g % ESTAGES;
                        mbar_wait(bar_empty + 8 * s, ((g / ESTAGES) & 1u) ^ 1u);
                        mbar_expect_tx(bar_full + 8 * s, ESTAGE_BYTES);
                        const int64_t woff = ((int64_t) h * ENC_NKT + kt) * TILE_ELEMS;
                        bulk_g2s(ring + s * ESTAGE_BYTES, G.wh_hi[dir] + woff, TILE_BYTES, bar_full + 8 * s);
                        bulk_g2s(ring + s * ESTAGE_BYTES + TILE_BYTES, G.wh_lo[dir] + woff, TILE_BYTES, bar_full + 8 * s);
                    }
            }
        }
        return;
    }
    reg_alloc<LSTM_CONS_REGS>();
    const int wg = warp >> 2, q = lane & 3;
    const int r128 = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * (q & 1);      // row of this lane's cells
    const int row = mt * BM + r128;
    const bool valid = row < G.M, odd_u = q >> 1;
    const float inv_s = G.inv_scale[dir];
    float4 *const cl = reinterpret_cast<float4 *>(G.c[dir] + c_index(q >> 1, row));   // this lane's first four cells
    uint32_t g = 0;
    float acc0[64], acc1[64], c0[16], c1[16];

    // the epilogue targets of half h of step t: units 32 h .. 32 h + 31 are operand k-tile h of the step (slice k-tile
    // 4 dir + h / 2, chunks 2 (h & 1), + 1)
    auto epi_of = [&](int t, int h) {
        const int tt = dir ? G.T - 1 - t : t;
        EncEpi E;
        E.sb = sbias + h * (PBN / 2) + 2 * q;
        E.cp = cl + h * 1024;
        E.yw = Q8 ? nullptr : (odd_u ? G.y_lo : G.y_hi) + (int64_t) mt * G.y_mt_stride + (int64_t) (tt * 16 + dir * 8 + h) * TILE_ELEMS + r128 * 8;
        E.qw = Q8 ? (odd_u ? G.q0 : G.q1) + mt * G.q_mt_stride + (int64_t) (tt * 8 + dir * 4 + (h >> 1)) * QTILE_BYTES + (h & 1) * 4096 + r128 * 16
                  : nullptr;
        E.yf = G.y_f32 ? G.y_f32 + (int64_t) row * G.ldy + (int64_t) tt * 512 + dir * 256 + h * 32 : nullptr;
        E.hs = hbuf + ((uint32_t) t & 1u) * EH_BYTES + h * TILE_BYTES + r128 * 16;
        return E;
    };
    auto release = [&](uint32_t gi) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * (gi % ESTAGES));
    };

    // Half h of step t into acc; the epilogue of the half before it (step t, h - 1, or step t - 1, 7) from accp / cp_ in
    // slices under its k-tiles 1-8.  ODD: h is odd (acc1), so the two sets are compile-time arrays in both calls.
    auto half = [&](auto odd_tag, int t, int h, float(&acc)[64], float(&cn)[16], float(&accp)[64], float(&cp_)[16]) {
        constexpr bool ODD = decltype(odd_tag)::value;
        const bool has_prev = ODD || t > 0 || h > 0;
        const EncEpi E = has_prev ? epi_of(h > 0 ? t : t - 1, h > 0 ? h - 1 : 7) : EncEpi{};
#ifdef PB_LSTM_TRACE
        const int tc0 = ((warp * G.T + t) * 8 + h) * 4;
#endif
        LSTM_STAMP(tc0);
        // this half's cell states, in flight during its k-loop
        {
            float4 *p = cl + h * 1024;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const float4 v = valid ? __ldcg(p + k * 256) : make_float4(0.f, 0.f, 0.f, 0.f);
                cn[4 * k] = v.x; cn[4 * k + 1] = v.y; cn[4 * k + 2] = v.z; cn[4 * k + 3] = v.w;
            }
        }
#pragma unroll
        for (int i = 0; i < 64; i++) acc[i] = 0.f;
        const uint32_t xa = xbuf + ((uint32_t) t & 1u) * TILE_BYTES + (uint32_t) wg * 1024;
        const uint32_t ha = hbuf + ((uint32_t) (t - 1) & 1u) * EH_BYTES + (uint32_t) wg * 1024;
        // k-tile 0: the step's image k-tile
        if (!ODD && h == 0) mbar_wait(bar_xfull + 8 * (t & 1), ((uint32_t) t >> 1) & 1u);
        mbar_wait(bar_full + 8 * (g % ESTAGES), (g / ESTAGES) & 1u);
        LSTM_STAMP(tc0 + 1);
        enc_ktile(acc, xa, ring + (g % ESTAGES) * ESTAGE_BYTES);
        wg_wait<1>();                                       // the previous half's accumulators are complete
        if (g > 0) release(g - 1);
        if (!ODD && h == 0 && t > 0) {                      // every group of step t - 1 is complete: its image slot is free
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_xempty + 8 * ((t - 1) & 1));
        }
        g++;
        if (t == 0) {
            // step 0 has no h-part: the previous half's epilogue runs after the image k-tile
            LSTM_STAMP(tc0 + 2);
            if (has_prev) {
#pragma unroll
                for (int m = 0; m < 8; m++) enc_cells<Q8>(accp, cp_, m, E, inv_s, q, odd_u, valid);
            }
            if (ODD && h == 7) enc_publish_h(wg);
        } else {
#pragma unroll
            for (int kt = 1; kt < ENC_NKT; kt++) {
                if (!ODD && kt == ENC_NKT - 1 && h == 0) {
                    // h k-tile 7 is the previous half's output: finish its epilogue and publish it first
                    enc_cells<Q8>(accp, cp_, 7, E, inv_s, q, odd_u, valid);
                    LSTM_STAMP(256 * G.T + (warp * G.T + t) * 2);
                    enc_publish_h(wg);
                    LSTM_STAMP(256 * G.T + (warp * G.T + t) * 2 + 1);
                }
                mbar_wait(bar_full + 8 * (g % ESTAGES), (g / ESTAGES) & 1u);
                enc_ktile(acc, ha + (kt - 1) * TILE_BYTES, ring + (g % ESTAGES) * ESTAGE_BYTES);
                if (kt == ENC_NKT - 1) LSTM_STAMP(tc0 + 2);
                if (ODD || kt < ENC_NKT - 1 || h > 0) enc_cells<Q8>(accp, cp_, kt - 1, E, inv_s, q, odd_u, valid);
                // h k-tiles 0-6 of the next step (halves 0-6) are written
                if (ODD && kt == ENC_NKT - 1 && h == 7) enc_publish_h(wg);
                wg_wait<1>();
                release(g - 1);
                g++;
            }
        }
        // no wgmma group stays in flight across the loop's back edge: ptxas serializes every wgmma of the kernel when one
        // does (it cannot follow wg_wait<1> around a loop), and this wait costs one k-tile's tail per half-tile pair
        if constexpr (ODD) wg_wait<0>();
        LSTM_STAMP(tc0 + 3);
    };

    for (int t = 0; t < G.T; t++) {
        for (int h = 0; h < 8; h += 2) {
            half(std::false_type{}, t, h, acc0, c0, acc1, c1);
            half(std::true_type{}, t, h + 1, acc1, c1, acc0, c0);
        }
    }
    // the last half tile's epilogue
    wg_wait<0>();
    release(g - 1);
    const EncEpi E = epi_of(G.T - 1, 7);
#pragma unroll
    for (int m = 0; m < 8; m++) enc_cells<Q8>(acc1, c1, m, E, inv_s, q, odd_u, valid);
#ifdef PB_LSTM_TRACE
    if (tr && threadIdx.x == 0) { tr[275 * G.T + 2] = trace_gtime(); tr[275 * G.T + 3] = trace_clock(); }
#endif
}

// ---------------------------------------------------------------- persistent LSTM decoder layer on int8 slices (variant, mode 2)
// k_lstm_layer's structure (one CTA per (direction, row tile) for all steps, one producer thread streaming whole tiles onto an
// mbarrier ring, h_t handed to the producer through bar_h) with int8-slice operands: K = [x (512) | h (256)] = 12 k-tiles of
// 64, 128-column gate tiles (32 units x 4 gates, 8 per step) so that the two int32 accumulators of a warpgroup take the 128
// registers one fp32 accumulator took.  Each step writes h_t only as int8 slices: they are the h-part of its own next step and,
// all 33 steps together, the A operand of linear_1 (k_gemm_q8).  Steps t0 .. t1 - 1 run in one launch: the cell state and h
// stay in HBM between launches, so launches of fewer steps are the cross-check of the in-kernel hand-off.
//
// The cell epilogue runs in a warpgroup of its own, under the next gate tile's k-loop.  The consumers' two accumulators leave
// no registers for a second set, so the hand-off goes through shared memory: once a tile's k-loop ends, the consumers fold
// hh / mix into fp32 pre-activations, fmaf(fmaf(hh, 256, mix), scale, bias), store them to the 64 KB staging buffer and go on
// to the next tile; epilogue thread r (0-127) runs the 32 cells of row r from there, writes the q1 / q0 slices (two 16 B
// chunks each), c and the optional y_f32, and after gate tile 7 publishes h_t to the producer.  Padding rows write nothing.
//
// Staging buffer: the pre-activation of (row r, unit j of the tile, gate g) sits at byte
//   j * 2048 + (r / 8) * 128 + ((r % 8) ^ 4 (j & 1)) * 16 + 4 g
// An epilogue thread reads a cell's four gates with one 16 B load, 8 consecutive rows of one unit filling one 128 B line.  A
// consumer lane stores two gates (8 B) of one unit and row; the XOR by unit parity puts the two units of a half-warp's
// store on disjoint banks, so each warp-wide store takes 2 wavefronts, the minimum for 256 B.
//
// Barriers (g: the launch's running k-tile count; n = 0 .. N - 1: its gate tiles, N = 8 (t1 - t0)):
//   bar_full[s]   mbarrier, count 1: the producer's arrive.expect_tx, completed by the bulk copies' bytes.  Every consumer
//                 warp waits on stage g % LQSTAGES with parity (g / LQSTAGES) & 1.
//   bar_empty[s]  mbarrier, count 8: lane 0 of each consumer warp, once the wgmma group that read the stage is complete.
//                 The producer waits before it refills the stage for k-tile g, with parity ((g / LQSTAGES) & 1) ^ 1.
//   bar_h         mbarrier, count 4: lane 0 of each epilogue warp after gate tile 7 of step t, its h_t slices written and
//                 __threadfence'd; that completes phase t - t0.  The producer waits on it with parity (t - t0) & 1, then
//                 fence.proxy.async, before the first h-part copy of step t + 1.  The launch's last phase has no waiter.
//   STAGED        named barrier 1, 384 threads: the 256 consumers bar.arrive once tile n is in the staging buffer; the 128
//                 epilogue threads bar.sync before reading it.  N times.
//   FREE          named barrier 2, 384 threads: the epilogue threads bar.arrive once they have read tile n, n < N - 1; the
//                 consumers bar.sync before storing tile n + 1.  N - 1 times, so no barrier is left half-arrived at exit.
// Each waits for the other before its next arrival, so neither named barrier ever has two generations in flight.  Every
// count and parity starts from the launch's first step, so a launch at t0 > 0 starts like the first one; c and the h
// slices of step t0 - 1 come from HBM, written by the previous launch.  The kernel ends when the epilogue warps have
// written the last tile.
struct LstmLayerQ {
    const int8_t *x1, *x0;             // input sequence slices (QSeq): tile (mt, tt, kt) at mt * q_mt_stride + (tt * 8 + kt) * QTILE_BYTES
    const int8_t *w1[2], *w0[2];       // per direction: [8 n-tiles][12 k-tiles][QTILE_BYTES]
    const float *bias[2];
    const float *col_scale[2];         // [1024] 256 / (32512 sw_n)
    float *c[2];                       // cell state per direction (c_index)
    int8_t *q1, *q0;                   // output sequence slices (QSeq); direction d -> k-tiles 4 d .. 4 d + 3
    int64_t q_mt_stride;               // bytes, the same for x and q
    float *y_f32;                      // optional fp32 copy [row][T][512]
    int64_t ldy;
    int M, n_mt, T, t0, t1;
#ifdef PB_LSTM_TRACE
    uint64_t *trace;                   // lstm_trace_words(T) stamps per launch, nullptr: none
#endif
};

template <int NS>
__device__ __forceinline__ void load_stage_q(uint32_t smem_base, uint32_t bar_full, uint32_t bar_empty, uint32_t g, const int8_t *a1,
                                             const int8_t *a0, const int8_t *w1, const int8_t *w0) {
    const uint32_t s = g % NS, ph = (g / NS) & 1u;
    mbar_wait(bar_empty + 8 * s, ph ^ 1u);
    const uint32_t st = smem_base + s * QSTAGE_BYTES;
    mbar_expect_tx(bar_full + 8 * s, QSTAGE_BYTES);
    bulk_g2s(st, a1, QTILE_BYTES, bar_full + 8 * s);
    bulk_g2s(st + QTILE_BYTES, a0, QTILE_BYTES, bar_full + 8 * s);
    bulk_g2s(st + 2 * QTILE_BYTES, w1, QTILE_BYTES, bar_full + 8 * s);
    bulk_g2s(st + 3 * QTILE_BYTES, w0, QTILE_BYTES, bar_full + 8 * s);
}

__device__ __forceinline__ void named_arrive(int id, int threads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
__device__ __forceinline__ void named_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
constexpr int LQ_STAGED = 1, LQ_FREE = 2, LQ_HANDOFF_THREADS = 32 * LQ_PROD_WARP;   // named barriers of warps 0-11

__global__ void __launch_bounds__(LQ_THREADS, 1) k_lstm_layer_q8(LstmLayerQ G) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int PRE = LQSTAGES * QSTAGE_BYTES, BARS = PRE + QPRE_BYTES;
    constexpr int X_NKT = 8, W_NKT = 12, N_TILES = 8;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + BARS);
    float *sbias = reinterpret_cast<float *>(smem + BARS + 256);
    float *sscale = sbias + 1024;
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + LQSTAGES), bar_h = smem_u32(bars + 2 * LQSTAGES);
    const uint32_t smem_base = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.x / G.n_mt, mt = blockIdx.x % G.n_mt;
    const int n_tiles = (G.t1 - G.t0) * N_TILES;

    if (threadIdx.x == 0) {
        for (int s = 0; s < LQSTAGES; s++) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, CONS_WARPS); }
        mbar_init(bar_h, LQ_PROD_WARP - LQ_EPI_WARP);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < 1024; i += LQ_THREADS) { sbias[i] = G.bias[dir][i]; sscale[i] = G.col_scale[dir][i]; }
#ifdef PB_LSTM_TRACE
    const int ts = blockIdx.x == 0 ? 0 : blockIdx.x == gridDim.x / 2 ? 1 : blockIdx.x == gridDim.x - 1 ? 2 : -1;
    uint64_t *const tr = G.trace && ts >= 0 ? G.trace + ts * lstm_trace_cta_words(G.T) : nullptr;
    if (tr && threadIdx.x == 0) { tr[275 * G.T] = trace_gtime(); tr[275 * G.T + 1] = trace_clock(); }
#endif
    __syncthreads();

    if (warp >= LQ_PROD_WARP) {
        reg_dealloc<LQ_PROD_REGS>();
        if (threadIdx.x == 32 * LQ_PROD_WARP) {
            uint32_t g = 0;
            for (int t = G.t0; t < G.t1; t++) {
                const int tt = dir ? G.T - 1 - t : t, tp = dir ? tt + 1 : tt - 1;
                const int nkt = X_NKT + (t > 0 ? W_NKT - X_NKT : 0);
                for (int nt = 0; nt < N_TILES; nt++) {
                    for (int kt = 0; kt < nkt; kt++, g++) {
                        const int8_t *a1, *a0;
                        if (kt < X_NKT) {
                            const int64_t off = (int64_t) mt * G.q_mt_stride + ((int64_t) tt * 8 + kt) * QTILE_BYTES;
                            a1 = G.x1 + off; a0 = G.x0 + off;
                        } else {
                            if (kt == X_NKT && nt == 0 && t > G.t0) {
                                // every epilogue warp has written its rows of h_{t-1}: make them visible to the bulk-copy engine
                                LSTM_STAMP(272 * G.T + t * 3);
                                mbar_wait(bar_h, (uint32_t) (t - G.t0 - 1) & 1u);
                                asm volatile("fence.proxy.async;" ::: "memory");
                                LSTM_STAMP(272 * G.T + t * 3 + 1);
                            }
                            const int64_t off = (int64_t) mt * G.q_mt_stride + ((int64_t) tp * 8 + dir * 4 + kt - X_NKT) * QTILE_BYTES;
                            a1 = G.q1 + off; a0 = G.q0 + off;
                        }
                        const int64_t woff = ((int64_t) nt * W_NKT + kt) * QTILE_BYTES;
                        load_stage_q<LQSTAGES>(smem_base, bar_full, bar_empty, g, a1, a0, G.w1[dir] + woff, G.w0[dir] + woff);
                        if (t > G.t0 && nt == 0 && kt == X_NKT) LSTM_STAMP(272 * G.T + t * 3 + 2);
                    }
                }
            }
        }
        return;
    }

    if (warp >= LQ_EPI_WARP) {
        reg_alloc<LQ_EPI_REGS>();
        const int r128 = threadIdx.x - 32 * LQ_EPI_WARP;                // the row of this thread's cells
        const int row = mt * BM + r128;
        const bool valid = row < G.M;
        // cells (nt * 32 + 8 a + b + 2 k, row) of c_index sit at cl[(nt * 4 + a) * 256 + 2 b], element k
        float4 *const cl = reinterpret_cast<float4 *>(G.c[dir] + c_index(0, row));
        const uint8_t *const srow = smem + PRE + (r128 >> 3) * 128;
        const int rx = r128 & 7;
        int n = 0;
        for (int t = G.t0; t < G.t1; t++) {
            const int tt = dir ? G.T - 1 - t : t;
            const int64_t qo = (int64_t) mt * G.q_mt_stride + (int64_t) (tt * 8 + dir * 4) * QTILE_BYTES + r128 * 16;
            float *yf = G.y_f32 ? G.y_f32 + (int64_t) row * G.ldy + (int64_t) tt * 512 + dir * 256 : nullptr;
            for (int nt = 0; nt < N_TILES; nt++, n++) {
#ifdef PB_LSTM_TRACE
                const int te0 = 275 * G.T + 4 + (((warp - LQ_EPI_WARP) * G.T + t) * 8 + nt) * 4;
#endif
                // the tile's 32 cell states, in flight while the consumers fold and stage
                float4 *cp = cl + nt * 4 * 256;
                float c[QN / 4];
#pragma unroll
                for (int a = 0; a < 4; a++)
#pragma unroll
                    for (int b = 0; b < 2; b++) {
                        const float4 v = valid ? __ldcg(cp + a * 256 + 2 * b) : make_float4(0.f, 0.f, 0.f, 0.f);
                        c[8 * a + b] = v.x; c[8 * a + b + 2] = v.y; c[8 * a + b + 4] = v.z; c[8 * a + b + 6] = v.w;
                    }
                LSTM_STAMP(te0);
                named_sync(LQ_STAGED, LQ_HANDOFF_THREADS);
                uint32_t w1[8], w0[8];
#pragma unroll
                for (int m = 0; m < 8; m++) {
                    // units 4 m .. 4 m + 3 of the tile: four independent cells, one word of each slice
                    int uq[4];
                    float h[4];
#pragma unroll
                    for (int e = 0; e < 4; e++) {
                        const int j = 4 * m + e;
                        const float4 gt = *reinterpret_cast<const float4 *>(srow + j * 2048 + ((rx ^ ((j & 1) << 2)) << 4));
                        const float cn = sigm(gt.y) * c[j] + sigm(gt.x) * tanh_fast(gt.z);
                        h[e] = sigm(gt.w) * tanh_fast(cn);
                        c[j] = cn;
                        uq[e] = qbias(h[e]);
                    }
                    w1[m] = qword(uq[0], uq[1], uq[2], uq[3], false);
                    w0[m] = qword(uq[0], uq[1], uq[2], uq[3], true);
                    if (yf && valid) *reinterpret_cast<float4 *>(yf + nt * (QN / 4) + 4 * m) = make_float4(h[0], h[1], h[2], h[3]);
                }
                if (n + 1 < n_tiles) named_arrive(LQ_FREE, LQ_HANDOFF_THREADS);
                if (valid) {
                    // units nt * 32 .. + 31 are chunks 2 (nt & 1), + 1 of slice k-tile 4 dir + nt / 2
                    const int64_t o = qo + (nt >> 1) * QTILE_BYTES + (nt & 1) * 2 * 2048;
                    __stwb(reinterpret_cast<uint4 *>(G.q1 + o), make_uint4(w1[0], w1[1], w1[2], w1[3]));
                    __stwb(reinterpret_cast<uint4 *>(G.q1 + o + 2048), make_uint4(w1[4], w1[5], w1[6], w1[7]));
                    __stwb(reinterpret_cast<uint4 *>(G.q0 + o), make_uint4(w0[0], w0[1], w0[2], w0[3]));
                    __stwb(reinterpret_cast<uint4 *>(G.q0 + o + 2048), make_uint4(w0[4], w0[5], w0[6], w0[7]));
#pragma unroll
                    for (int a = 0; a < 4; a++)
#pragma unroll
                        for (int b = 0; b < 2; b++)
                            cp[a * 256 + 2 * b] = make_float4(c[8 * a + b], c[8 * a + b + 2], c[8 * a + b + 4], c[8 * a + b + 6]);
                }
                LSTM_STAMP(te0 + 1);
            }
            // h_t of this warp's rows is complete (all eight gate tiles): publish it to the producer thread
            __threadfence();
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_h);
            LSTM_STAMP(275 * G.T + 4 + (((warp - LQ_EPI_WARP) * G.T + t) * 8 + 7) * 4 + 2);
        }
        return;
    }

    reg_alloc<LQ_CONS_REGS>();
    const int wg = warp >> 2, q = lane & 3;
    const int rA = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    // accumulator fragment of m64n128: [4 i + 2 h + e] is row rA + 8 h, column 8 i + 2 q + e = gate 2 (q & 1) + e of unit
    // 2 i + q / 2.  This lane's staging slot of (unit q / 2, row rA); unit 2 i + q / 2 and row rA + 8 h are i * 4096 + h * 128
    // bytes on (2 i is even, so the unit parity, and with it the XOR, is the lane's own).
    float *const sp = reinterpret_cast<float *>(smem + PRE + (q >> 1) * 2048 + (rA >> 3) * 128 + ((((lane >> 2) ^ ((q >> 1) << 2))) << 4) +
                                                (q & 1) * 8);
    uint32_t g = 0;
    int n = 0;
    int hh[64], mix[64];
    for (int t = G.t0; t < G.t1; t++) {
        const int nkt = X_NKT + (t > 0 ? W_NKT - X_NKT : 0);
        for (int nt = 0; nt < N_TILES; nt++, n++) {
#ifdef PB_LSTM_TRACE
            const int tc0 = ((warp * G.T + t) * 8 + nt) * 4;
#endif
            LSTM_STAMP(tc0);
#pragma unroll
            for (int i = 0; i < 64; i++) { hh[i] = 0; mix[i] = 0; }
            for (int kt = 0; kt < nkt; kt++, g++) {
                const uint32_t s = g % LQSTAGES, ph = (g / LQSTAGES) & 1u;
                mbar_wait(bar_full + 8 * s, ph);
                if (kt == 0) LSTM_STAMP(tc0 + 1);
                const uint32_t st = smem_base + s * QSTAGE_BYTES, a = st + (uint32_t) wg * 1024, b = st + 2 * QTILE_BYTES;
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < QK / 32; ks++) {
                    const uint64_t a1 = smem_desc(a + ks * 4096, 2048), a0 = smem_desc(a + QTILE_BYTES + ks * 4096, 2048);
                    const uint64_t w1 = smem_desc(b + ks * 4096, 2048), w0 = smem_desc(b + QTILE_BYTES + ks * 4096, 2048);
                    wgmma_q8(hh, a1, w1);
                    wgmma_q8(mix, a1, w0);
                    wgmma_q8(mix, a0, w1);
                }
                wg_commit();
                wg_wait<1>();
                if (kt > 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_empty + 8 * ((g - 1) % LQSTAGES));
                }
            }
            wg_wait<0>();
            LSTM_STAMP(tc0 + 2);
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8 * ((g - 1) % LQSTAGES));

            const float *sb = sbias + nt * QN + 2 * q, *ss = sscale + nt * QN + 2 * q;
            if (n > 0) named_sync(LQ_FREE, LQ_HANDOFF_THREADS);       // the epilogue warps have read tile n - 1
#pragma unroll
            for (int i = 0; i < QN / 8; i++) {
                const float2 bz = *reinterpret_cast<const float2 *>(sb + 8 * i), sz = *reinterpret_cast<const float2 *>(ss + 8 * i);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const float v0 = fmaf(fmaf((float) hh[4 * i + 2 * h], 256.f, (float) mix[4 * i + 2 * h]), sz.x, bz.x);
                    const float v1 = fmaf(fmaf((float) hh[4 * i + 2 * h + 1], 256.f, (float) mix[4 * i + 2 * h + 1]), sz.y, bz.y);
                    *reinterpret_cast<float2 *>(sp + i * 1024 + h * 32) = make_float2(v0, v1);
                }
            }
            LSTM_STAMP(tc0 + 3);
            named_arrive(LQ_STAGED, LQ_HANDOFF_THREADS);
        }
    }
#ifdef PB_LSTM_TRACE
    if (tr && threadIdx.x == 0) { tr[275 * G.T + 2] = trace_gtime(); tr[275 * G.T + 3] = trace_clock(); }
#endif
}

// ---------------------------------------------------------------- persistent GEMM on int8 slices (linear_1, mode 2)
// Y = SELU(A W^T + bias) with A in [-1, 1] held as QSeq slices (the decoder's h, all 33 steps, read in place) and W packed per
// output row like the decoder's gate rows.  k_tc_gemm_p's tile loop (one CTA per SM, static round-robin over 128 x 128
// output tiles, nt fastest so that CTAs running together share the A row tile) around k_lstm_layer_q8's k-loop: the
// producer thread streams a1, a0, w1, w0 of one 64-k tile per ring stage and runs ahead across tiles, so the next tile's
// operands arrive while the consumers apply the epilogue of the current one.  No split-K: a row's outputs do not depend on
// which other rows share its launch.  |acc_hh| <= K 127^2 and |acc_mix| <= 2 K 127 128 stay below 2^31 for K < 65,000.
struct GemmQ {
    const int8_t *a1, *a0;             // A slices: tile (mt, kt) at mt * a_mt_stride + kt * QTILE_BYTES
    int64_t a_mt_stride;               // bytes
    const int8_t *w1, *w0;             // [N / 128 n-tiles][nkt][QTILE_BYTES]
    const float *bias, *col_scale;     // [N]; col_scale 256 / (32512 sw_n)
    op_t *y_hi, *y_lo;                 // output operand tiles [mt][N / 32][TILE_ELEMS] (the next layer's A)
    float *y_f32;                      // optional fp32 copy [M][N]
    int M, N, n_mt, nkt;
};

__global__ void __launch_bounds__(PG_THREADS, 1) k_gemm_q8(GemmQ G) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + QSTAGES * QSTAGE_BYTES);
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + QSTAGES);
    const uint32_t smem_base = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_nt = G.N / QN, n_tiles = G.n_mt * n_nt;

    if (threadIdx.x == 0) {
        for (int s = 0; s < QSTAGES; s++) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, CONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == CONS_WARPS) {
        if (lane == 0) {
            uint32_t g = 0;                                   // running k-tile counter across tiles
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                const int nt = tile % n_nt, mt = tile / n_nt;
                const int64_t aoff = (int64_t) mt * G.a_mt_stride, woff = (int64_t) nt * G.nkt * QTILE_BYTES;
                for (int kt = 0; kt < G.nkt; kt++, g++) {
                    const int64_t ko = (int64_t) kt * QTILE_BYTES;
                    load_stage_q<QSTAGES>(smem_base, bar_full, bar_empty, g, G.a1 + aoff + ko, G.a0 + aoff + ko, G.w1 + woff + ko, G.w0 + woff + ko);
                }
            }
        }
        return;
    }
    const int wg = warp >> 2, q = lane & 3;
    const int rA = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    uint32_t g = 0;
    int hh[64], mix[64];
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int nt = tile % n_nt, mt = tile / n_nt;
#pragma unroll
        for (int i = 0; i < 64; i++) { hh[i] = 0; mix[i] = 0; }
        for (int kt = 0; kt < G.nkt; kt++, g++) {
            const uint32_t s = g % QSTAGES, ph = (g / QSTAGES) & 1u;
            mbar_wait(bar_full + 8 * s, ph);
            const uint32_t st = smem_base + s * QSTAGE_BYTES, a = st + (uint32_t) wg * 1024, b = st + 2 * QTILE_BYTES;
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < QK / 32; ks++) {
                const uint64_t a1 = smem_desc(a + ks * 4096, 2048), a0 = smem_desc(a + QTILE_BYTES + ks * 4096, 2048);
                const uint64_t w1 = smem_desc(b + ks * 4096, 2048), w0 = smem_desc(b + QTILE_BYTES + ks * 4096, 2048);
                wgmma_q8(hh, a1, w1);
                wgmma_q8(mix, a1, w0);
                wgmma_q8(mix, a0, w1);
            }
            wg_commit();
            wg_wait<1>();
            if (kt > 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_empty + 8 * ((g - 1) % QSTAGES));
            }
        }
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * ((g - 1) % QSTAGES));
        // accumulator fragment of m64n128: [4 i + e] is row rA + 8 (e >> 1), column 8 i + 2 q + (e & 1)
#pragma unroll
        for (int i = 0; i < QN / 8; i++) {
            const int col = nt * QN + 8 * i + 2 * q;
            const float2 bz = __ldg(reinterpret_cast<const float2 *>(G.bias + col));
            const float2 sz = __ldg(reinterpret_cast<const float2 *>(G.col_scale + col));
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int r128 = rA + 8 * h, row = mt * BM + r128;
                const int e = 4 * i + 2 * h;
                const float v0 = selu(fmaf(fmaf((float) hh[e], 256.f, (float) mix[e]), sz.x, bz.x));
                const float v1 = selu(fmaf(fmaf((float) hh[e + 1], 256.f, (float) mix[e + 1]), sz.y, bz.y));
                if (row < G.M) {
                    uint32_t hi, lo;
                    split2(v0, v1, hi, lo);
                    const int64_t o = (int64_t) mt * (G.N / BK) * TILE_ELEMS + tile_off(col, r128);
                    *reinterpret_cast<uint32_t *>(G.y_hi + o) = hi;
                    *reinterpret_cast<uint32_t *>(G.y_lo + o) = lo;
                    if (G.y_f32) *reinterpret_cast<float2 *>(G.y_f32 + (int64_t) row * G.N + col) = make_float2(v0, v1);
                }
            }
        }
    }
}

// ---------------------------------------------------------------- persistent GRU layer kernel (polish)
// All 100 time steps of one bidirectional GRU layer of one window in ONE launch, one CTA per (direction, row tile): the
// CTA computes both 256-column gate tiles (128 hidden units x {r, z, n_x, n_h}) of every step, so h never has to be
// exchanged with another CTA.  h_t goes out as operand tiles of the layer's output sequence and comes back through the
// bulk-copy ring as the h-part of step t+1; the previous hidden values of the cell update are re-read from those tiles
// (L2).  Step 0 takes h0.
struct GruWin {
    const op_t *x_hi, *x_lo;           // input sequence operand [mt][100][x_kt] tiles (x_lo == nullptr: exact input)
    int x_kt;
    const op_t *h0_hi[2], *h0_lo[2];   // initial state tiles per direction (4 k-tiles per row tile)
    int64_t h0_mt_stride;
    const op_t *w_hi[2], *w_lo[2];     // per direction: [nt(2)][x_kt + 4][WTILE_ELEMS]
    const float *bias[2];
    float inv_scale[2];                // 1 / s of each direction's packed weight
    op_t *y_hi, *y_lo;                 // output sequence operand [mt][100][8] tiles
    int M, n_mt, T;
    int lo_x, lo_h;                    // 1 = execute the a_lo x w_hi product of the x-part / h-part
};

__global__ void __launch_bounds__(PG_THREADS, 1) k_gru_layer(GruWin G) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + PSTAGES * PSTAGE_BYTES);
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + PSTAGES), bar_h = smem_u32(bars + 2 * PSTAGES);
    const uint32_t smem_base = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.x / G.n_mt, mt = blockIdx.x % G.n_mt;
    const int nkt = G.x_kt + 4;
    const int64_t seq_stride = (int64_t) G.T * 8 * TILE_ELEMS;

    if (threadIdx.x == 0) {
        for (int s = 0; s < PSTAGES; s++) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, CONS_WARPS); }
        mbar_init(bar_h, CONS_WARPS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == CONS_WARPS) {
        if (lane == 0) {
            uint32_t g = 0;
            for (int t = 0; t < G.T; t++) {
                const int tt = dir ? G.T - 1 - t : t, tp = dir ? tt + 1 : tt - 1;
                for (int nt = 0; nt < 2; nt++) {
                    for (int kt = 0; kt < nkt; kt++, g++) {
                        const op_t *a_hi, *a_lo;
                        if (kt < G.x_kt) {
                            const int64_t off = ((int64_t) (mt * G.T + tt) * G.x_kt + kt) * TILE_ELEMS;
                            a_hi = G.x_hi + off; a_lo = (G.x_lo && G.lo_x) ? G.x_lo + off : nullptr;
                        } else {
                            const int kk = kt - G.x_kt;
                            if (t == 0) {
                                const int64_t off = (int64_t) mt * G.h0_mt_stride + (int64_t) kk * TILE_ELEMS;
                                a_hi = G.h0_hi[dir] + off; a_lo = G.lo_h ? G.h0_lo[dir] + off : nullptr;
                            } else {
                                if (kk == 0 && nt == 0) {
                                    mbar_wait(bar_h, (uint32_t) (t - 1) & 1u);      // every consumer warp has written its part of h_{t-1}
                                    asm volatile("fence.proxy.async;" ::: "memory");
                                }
                                const int64_t off = (int64_t) mt * seq_stride + ((int64_t) tp * 8 + dir * 4 + kk) * TILE_ELEMS;
                                a_hi = G.y_hi + off; a_lo = G.lo_h ? G.y_lo + off : nullptr;
                            }
                        }
                        const int64_t woff = ((int64_t) nt * nkt + kt) * WTILE_ELEMS;
                        load_stage(smem_base, bar_full, bar_empty, g, a_hi, a_lo, G.w_hi[dir] + woff, G.w_lo[dir] + woff);
                    }
                }
            }
        }
        return;
    }
    const int wg = warp >> 2, q = lane & 3;
    const int r128 = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * (q & 1);
    const bool valid = mt * BM + r128 < G.M;
    const float *bias = G.bias[dir];
    const float inv_s = G.inv_scale[dir];
    const bool lo_x = G.x_lo != nullptr && G.lo_x != 0, lo_h = G.lo_h != 0;
    uint32_t g = 0;
    float acc[128];
    for (int t = 0; t < G.T; t++) {
        const int tt = dir ? G.T - 1 - t : t, tp = dir ? tt + 1 : tt - 1;
        // previous hidden state: h0, or the units this warp wrote in step t-1
        const op_t *hp_hi = t == 0 ? G.h0_hi[dir] + (int64_t) mt * G.h0_mt_stride : G.y_hi + (int64_t) mt * seq_stride + ((int64_t) tp * 8 + dir * 4) * TILE_ELEMS;
        const op_t *hp_lo = t == 0 ? G.h0_lo[dir] + (int64_t) mt * G.h0_mt_stride : G.y_lo + (int64_t) mt * seq_stride + ((int64_t) tp * 8 + dir * 4) * TILE_ELEMS;
        const int64_t y0 = (int64_t) mt * seq_stride + ((int64_t) tt * 8 + dir * 4) * TILE_ELEMS;
        for (int nt = 0; nt < 2; nt++) {
            mma_tile(acc, smem_base, bar_full, bar_empty, g, nkt, G.x_kt, lo_x, lo_h, wg, lane);
#pragma unroll
            for (int i = 0; i < PBN / 8; i++) {
                const int j = nt * (PBN / 4) + 2 * i + (q >> 1);
                float gt[4];
                gates4(acc, i, __ldg(reinterpret_cast<const float2 *>(bias + nt * PBN + 8 * i + 2 * q)), inv_s, q, gt);
                const float hp = valid ? load_h(hp_hi, hp_lo, tile_off(j, r128)) : 0.f;
                const float r = sigm(gt[0]), z = sigm(gt[1]);
                const float n = tanh_fast(gt[2] + r * gt[3]);
                store_h((1.0f - z) * n + z * hp, valid && !(q & 2), G.y_hi, G.y_lo, y0 + tile_off(j, r128), nullptr);
            }
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_h);
    }
}

// ---------------------------------------------------------------- operand preparation kernels
// int8 images [B][T][F] -> tiled operand [mt][T][1 k-tile] (hi only; |v| <= 128 is exact in the operand type)
__global__ void k_tc_pack_images(const int8_t *__restrict__ img, op_t *__restrict__ op, int64_t B, int T, int F) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;     // one thread per (row, t, kc)
    const int64_t total = ceil_div(B, 128) * 128 * T * 4;
    if (i >= total) return;
    const int kc = (int) (i & 3);
    const int64_t rt = i >> 2;
    const int t = (int) (rt % T);
    const int64_t row = rt / T;
    uint32_t w[4] = {0, 0, 0, 0};
    if (row < B) {
#pragma unroll
        for (int e = 0; e < 8; e++) {
            const int k = kc * 8 + e;
            const float v = (k < F) ? (float) img[(row * T + t) * F + k] : 0.f;
            w[e >> 1] |= (uint32_t) op_bits(v) << (16 * (e & 1));
        }
    }
    const int64_t o = ((row >> 7) * T + t) * TILE_ELEMS + kc * 1024 + (row & 127) * 8;
    *reinterpret_cast<uint4 *>(op + o) = make_uint4(w[0], w[1], w[2], w[3]);
}

}  // namespace tc
}  // namespace pb
