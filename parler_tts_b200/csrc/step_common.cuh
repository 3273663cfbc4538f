// step_common.cuh -- what the two decode-step kernels (step.cu, step2.cu) must compute identically, written once: they promise
// the same bits, so the embedding sum and the decode attention's arguments are not kept in two copies.
#pragma once
#include "attn_core.cuh"
#include "common.cuh"
#include "sample_core.cuh"
#include "step.h"

namespace ptts {

// Input embedding of batch row `row`, column `col`, for the token fed at cache position `pos`: the K codebook embeddings of the
// row's current ids added left to right with a bf16 rounding after each add, then the position embedding (models without
// rope).  Codebooks go in groups of 8: the loads of a group are in flight together, and the group's values are all that is live.
__device__ __forceinline__ float embed_value(const StepParams& p, int row, int col, int pos) {
  const bf16* tables = reinterpret_cast<const bf16*>(p.blob + p.lay.embed);
  float v = 0.f;
#pragma unroll 1
  for (int k0 = 0; k0 < p.K; k0 += 8) {
    float ev[8];
#pragma unroll
    for (int k = 0; k < 8; k++)
      if (k0 + k < p.K) ev[k] = __bfloat162float(tables[((size_t)(k0 + k) * (p.V + 1) + p.sa.cur_ids[row * p.K + k0 + k]) * p.H + col]);
#pragma unroll
    for (int k = 0; k < 8; k++)
      if (k0 + k < p.K) v = (k0 + k == 0) ? ev[k] : DT<bf16>::rnd(v + ev[k]);
  }
  if (!p.rope) v = DT<bf16>::rnd(v + __bfloat162float(reinterpret_cast<const bf16*>(p.blob + p.lay.pos)[(size_t)pos * p.H + col]));
  return v;
}

// Decode attention of layer l at cache position pos: self-attention over the K/V cache (the call also appends this step's K/V
// row to it) or cross-attention over the cached encoder K/V.  The caller sets where the query, this step's K/V (self only) and
// the output live: q / ldq, knew / vnew / ldkv / k_col0 / v_col0, out / ldo.
__device__ __forceinline__ AttnArgs decode_attn_args(const StepParams& p, int l, int pos, bool cross) {
  AttnArgs a{};
  a.ctrl = nullptr; a.B = p.B; a.nh = p.nh; a.q_len = 1;
  a.past_from_ctrl = 0; a.past_len = pos; a.prefix = p.P;
  a.rope = p.rope; a.rope_cos = p.blob + p.lay.rope_cos; a.rope_sin = p.blob + p.lay.rope_sin; a.scale = p.scale;
  if (!cross) {
    char* kc = p.self_kv + p.self_layer_stride * l;
    a.kcache = kc; a.vcache = kc + (size_t)p.B * p.nkv * p.Tmax * HD * 2;
    a.kv_b_stride = (int64_t)p.nkv * p.Tmax * HD; a.kv_h_stride = (int64_t)p.Tmax * HD; a.kv_t_stride = HD; a.kv_b_div = 1;
    a.key_mask = p.prompt_mask; a.mask_len = p.P; a.mask_ld = p.P;
    a.nkv = p.nkv; a.cross = 0; a.kv_len = 0; a.kv_capacity = p.Tmax;
  } else {
    char* ck = p.cross_kv + p.cross_layer_stride * l;
    a.kcache = ck; a.vcache = ck + (size_t)(p.B / p.takes) * p.nckv * p.S * HD * 2;   // one K/V item per description
    a.kv_b_stride = (int64_t)p.nckv * p.S * HD; a.kv_h_stride = (int64_t)p.S * HD; a.kv_t_stride = HD; a.kv_b_div = p.takes;
    a.key_mask = p.enc_mask; a.mask_len = p.S; a.mask_ld = p.S;
    a.nkv = p.nckv; a.cross = 1; a.kv_len = p.S; a.kv_capacity = p.S;
  }
  return a;
}

// Sampling phase: logits -> next token of every (utterance, codebook) row, one CTA per row (sample_core.cuh).  Not inlined: the
// sampler's registers then do not add to the decode phases' in the kernel's allocation.
template <int ITEMS>
__device__ __noinline__ void sample_phase(const SampleArgs& sa, const ptts_gen_params& gp, int BK, int cur_len) {
  sample_all_rows_cta<ITEMS>(sa, gp, (int)blockIdx.x, (int)gridDim.x, BK, cur_len);
}

}  // namespace ptts
