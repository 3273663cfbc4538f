// ln_stats.cuh -- LayerNorm folded into the following linear layer (bf16 model dtype).
//
// Reference: y = Linear(LayerNorm(x)) (modeling_parler_tts.py:1020-1023, :1040-1041, :1059-1060, :1632 + :1917-1920).
// With LN(x)_k = (x_k - mu) * r * g_k + b_k:
//     y_n = r * ( sum_k x_k W'_nk  -  mu * c1_n ) + c2_n,   W' = bf16(g_k W_nk),  c1_n = sum_k W'_nk,  c2_n = sum_k b_k W_nk
// W', c1, c2 are produced ONCE at load (ptts_decoder_finalize); at run time the GEMM consumes the RAW activation tile and
// only the per-row (mu, r) are needed -- one vectorised pass over the staged tile instead of a three-pass in-place
// normalisation that every CTA of the step kernel (one per SM) would repeat in every LN-fused GEMM phase.
// The per-row statistics ride on the tensor cores: with the A fragments of an m16 x k16 slab already in registers
// (ldmatrix), the SAME registers are valid B fragments of the slab's own transpose, so
//     D[r][c] += sum_k x[r,k] * x[c,k]      (two m16n8k16 per slab; the diagonal is sum_k x[r,k]^2)
//     D[r][*] += sum_k x[r,k] * 1           (one m16n8k16 against a fragment of bf16 ones)
// i.e. 12 mma per 32-row x 32-column slab instead of ~500 scalar FP instructions per thread in every LN-fused GEMM phase.  Products of bf16 are exact in fp32 and the accumulation is fp32:
// mean = S1/K, var = S2/K - mean^2 (un-shifted; relative error of var ~ 1e-6 * (1 + mean^2/var), far below the bf16
// resolution of the surrounding arithmetic for any realistic residual stream).
// Numerics vs the reference: the normalised activations are no longer rounded to bf16 before the GEMM and gamma is
// rounded into the weights instead; both effects are at the bf16 resolution of the reference's own arithmetic.
// The same functions are used by linear_bf16_kernel (gemm.cu) and decode_step_kernel (step.cu) with the same K split
// over warps and the same fixed reduction order: the two paths stay bit-identical.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace ptts {

// accumulators of one warp for a 32-row tile (two m16 tiles)
struct RowStatFrag {
  float s1[2][4];      // [mt]: D[r][*] = sum_k x[r,k]
  float sq[2][2][4];   // [mt][h]: D[r][c] = x_r . x_c for c in rows 8h..8h+7 of the same m-tile
};

__device__ __forceinline__ void row_stat_zero(RowStatFrag& st) {
#pragma unroll
  for (int mt = 0; mt < 2; mt++)
#pragma unroll
    for (int e = 0; e < 4; e++) { st.s1[mt][e] = 0.f; st.sq[mt][0][e] = 0.f; st.sq[mt][1][e] = 0.f; }
}

// one m16 x k16 slab (a = its ldmatrix.x4 A fragment: rows g | g+8, k low | high)
__device__ __forceinline__ void row_stat_mma(RowStatFrag& st, int mt, const uint32_t (&a)[4]) {
  constexpr uint32_t ONES = 0x3F803F80u;  // bf16x2 (1, 1)
  mma_bf16_16816(st.s1[mt], a, ONES, ONES);
  mma_bf16_16816(st.sq[mt][0], a, a[0], a[2]);  // B[k][n] = x[row n][k], rows 0-7 of the m-tile
  mma_bf16_16816(st.sq[mt][1], a, a[1], a[3]);  // rows 8-15
}

// one warp's pass over its slabs kt = warp, warp + 8, ... of a staged [16 * MT][kt_count * 32] tile (row pitch in elements)
template <int MT = 2>
__device__ __forceinline__ void row_stat_pass(RowStatFrag& st, const bf16* xs, int pitch, int kt_count, int warp, int lane) {
  const int lrow = (lane & 7) + ((lane >> 3) & 1) * 8, lcol = (lane >> 4) * 8;
  for (int kt = warp; kt < kt_count; kt += 8) {
#pragma unroll
    for (int mt = 0; mt < MT; mt++)
#pragma unroll
      for (int j = 0; j < 2; j++) {
        uint32_t a[4];
        ldmatrix_x4(a, xs + (size_t)(mt * 16 + lrow) * pitch + kt * 32 + j * 16 + lcol);
        row_stat_mma(st, mt, a);
      }
  }
}

// part: shared float[8 warps][32 rows][2] -- this warp's partial (S1, S2) of every row (rows 0..16*MT-1 are written)
template <int MT = 2>
__device__ __forceinline__ void row_stat_store(const RowStatFrag& st, float* part, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < MT; mt++) {
    float* pr = part + ((size_t)warp * 32 + mt * 16 + g) * 2;
    if (t == 0) { pr[0] = st.s1[mt][0]; pr[16] = st.s1[mt][2]; }
    if (t == (g >> 1)) {  // the thread holding the diagonal entries (g, g) and (g+8, g+8)
      pr[1] = (g & 1) ? st.sq[mt][0][1] : st.sq[mt][0][0];
      pr[17] = (g & 1) ? st.sq[mt][1][3] : st.sq[mt][1][2];
    }
  }
}

// threads 0..31 (one row each): fixed-order sum over the 8 warps -> stats[2r] = mean, stats[2r+1] = rstd
__device__ __forceinline__ void row_stat_finalize(const float* part, int K, int M, float eps, float* stats) {
  const int r = threadIdx.x;
  if (r < 32 && r < M) {
    float S1 = 0.f, S2 = 0.f;
#pragma unroll
    for (int w = 0; w < 8; w++) { S1 += part[((size_t)w * 32 + r) * 2]; S2 += part[((size_t)w * 32 + r) * 2 + 1]; }
    const float mean = S1 / (float)K;
    stats[2 * r] = mean;
    stats[2 * r + 1] = rsqrtf(fmaxf(S2 / (float)K - mean * mean, 0.f) + eps);
  }
}

}  // namespace ptts
