// probe.cu -- generate()'s and forward()'s output_attentions / output_hidden_states, written from inside run_forward.
//
// attention_probs_kernel: one layer's self- or cross-attention weights by the reference's EAGER definition (ParlerTTSAttention
// .forward, modeling_parler_tts.py:494-584), which is what it returns when asked for them: q = dtype(q_proj(x)) * scaling (exact for
// head_dim 64) with RoPE in the model dtype, scores = dtype(q . k^T) plus the additive finfo.min mask, softmax in fp32 rounded to the
// model dtype.  A row whose keys are all masked is uniform over all T_kv keys (every score is finfo.min there).  The q and K it
// reads are the ones the session's attention kernels read (the QKV output / W.qc, the swizzled caches); the tokens stay on the
// restated attention, so the weights cannot change them.
//
// One CTA per (batch row, head, tile of QT query rows): the QT queries stay in shared memory, every thread takes one key at a time
// (its 128-byte row is read once per CTA; self-attention stops at the tile's last query position) and keeps the rounded scores of
// the tile's rows in shared memory; then one warp per row takes the max / sum and writes the row.  The dot products are a scalar
// sweep: at decode (one query row) the kernel is bound by the K rows it reads and the row it writes, while a long teacher-forced
// prefill is compute-bound here (a tensor-core q.k^T is not written yet).  probe_rows_kernel copies residual-stream rows into the
// hidden-state output, or applies the final LayerNorm (fp32 statistics, the unfolded fp32 gamma / beta of the blob) for the last
// entry.
//
// Both take an optional decode window: with ctrl set (the decode graph), the step is ctrl->cur_len - n0 and a step outside
// [first_step, first_step + n_steps) writes nothing, like a finished generation (ctrl->active == 0).
#include <cfloat>

#include "attn_core.cuh"
#include "common.cuh"
#include "kernels.h"

namespace ptts {

// the decode window: the output slot of this step (nullptr: not recorded), and cur_len through *cur_len
template <typename P>
__device__ __forceinline__ char* probe_slot(const P& a, char* base, int* cur_len) {
  if (a.ctrl == nullptr) return base;
  if (a.ctrl->active == 0) return nullptr;
  const int cl = a.ctrl->cur_len;
  const int slot = cl - a.n0 - a.first_step;
  if (slot < 0 || slot >= a.n_steps) return nullptr;
  *cur_len = cl;
  return base + (int64_t)slot * a.step_bytes;
}

template <typename T, int QT>
__global__ void __launch_bounds__(QT * 32) attention_probs_kernel(AttnProbeArgs a) {
  extern __shared__ __align__(16) float smp[];
  float* qs = smp;               // [QT][64] scaled, rotated queries (model-dtype values)
  float* sc = smp + QT * HD;     // [QT][T_kv] rounded scores; -inf marks a masked key
  const int b = blockIdx.z, h = blockIdx.y, j0 = blockIdx.x * QT;
  int cur_len = 0;
  char* out = probe_slot(a, reinterpret_cast<char*>(a.out), &cur_len);
  if (out == nullptr) return;
  const int pos0 = a.ctrl != nullptr ? a.prefix + cur_len - 1 : a.pos0;   // position of query row 0
  const int T_kv = a.cross ? a.kv_len : (a.ctrl != nullptr ? pos0 + 1 : a.kv_len);
  const int kvh = h / (a.nh / a.nkv);
  const int kvb = b / a.kv_b_div;   // batch index of the K rows and the key mask
  const T* kc = reinterpret_cast<const T*>(a.kcache) + (size_t)kvb * a.kv_b_stride + (size_t)kvh * a.kv_h_stride;
  const T* rope_cos = reinterpret_cast<const T*>(a.rope_cos);
  const T* rope_sin = reinterpret_cast<const T*>(a.rope_sin);
  const int* km = a.key_mask ? a.key_mask + (size_t)kvb * a.mask_ld : nullptr;
  const int nq = min(QT, a.q_len - j0);

  for (int i = threadIdx.x; i < QT * HD; i += blockDim.x) {
    const int r = i / HD, d = i % HD;
    float x = 0.f;
    if (r < nq) {
      const T* src = reinterpret_cast<const T*>(a.q) + ((size_t)b * a.q_len + j0 + r) * a.ldq + a.q_col0 + (size_t)h * HD;
      x = DT<T>::to_f(src[d]);
      if (a.rope) {
        const int pos = pos0 + j0 + r;
        const float xp = DT<T>::to_f(src[d < HD / 2 ? d + HD / 2 : d - HD / 2]);
        x = rope_elem<T>(x, xp, d, rope_cos + (size_t)pos * HD, rope_sin + (size_t)pos * HD);
      }
      x = DT<T>::rnd(x * a.scale);
    }
    qs[i] = x;
  }
  __syncthreads();

  // self-attention: keys past the tile's last query position are masked for every row of it (no dot products for them)
  const int t_end = a.cross ? T_kv : min(T_kv, pos0 + j0 + nq);
  for (int t = t_end + threadIdx.x; t < T_kv; t += blockDim.x)
#pragma unroll
    for (int r = 0; r < QT; r++) sc[(size_t)r * T_kv + t] = -INFINITY;
  for (int t = threadIdx.x; t < t_end; t += blockDim.x) {
    float acc[QT];
#pragma unroll
    for (int r = 0; r < QT; r++) acc[r] = 0.f;
    const T* krow = kc + (size_t)t * HD;
#pragma unroll
    for (int c = 0; c < HD / 8; c++) {
      float kv[8];
      load8(krow + kv_swz(t, 8 * c), kv);   // dims 8c .. 8c + 7 of key t
#pragma unroll
      for (int r = 0; r < QT; r++)
#pragma unroll
        for (int e = 0; e < 8; e++) acc[r] = fmaf(qs[r * HD + 8 * c + e], kv[e], acc[r]);
    }
    const bool pad = km != nullptr && t < a.mask_len && km[t] == 0;
#pragma unroll
    for (int r = 0; r < QT; r++) {
      const bool vis = !pad && (a.cross || t <= pos0 + j0 + r);
      sc[(size_t)r * T_kv + t] = vis ? DT<T>::rnd(acc[r]) : -INFINITY;
    }
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp >= nq) return;
  const float* row = sc + (size_t)warp * T_kv;
  T* o = reinterpret_cast<T*>(out) + (size_t)b * a.out_b + (size_t)h * a.out_h + (size_t)(j0 + warp) * a.out_q;
  float m = -INFINITY;
  for (int t = lane; t < T_kv; t += 32) m = fmaxf(m, row[t]);
  m = warp_max(m);
  if (m == -INFINITY) {   // every key masked: the scores are all finfo.min, the softmax is uniform
    const T u = DT<T>::from_f(1.0f / (float)T_kv);
    for (int t = lane; t < T_kv; t += 32) o[t] = u;
    return;
  }
  float l = 0.f;
  for (int t = lane; t < T_kv; t += 32) l += expf(row[t] - m);
  l = warp_sum(l);
  for (int t = lane; t < T_kv; t += 32) __stcs(o + t, DT<T>::from_f(expf(row[t] - m) / l));
}

// rows [rows][H] -> the output slot; ln_w != nullptr: LayerNorm (two-pass fp32 statistics) instead of a copy.  One warp per row.
template <typename T>
__global__ void __launch_bounds__(256) probe_rows_kernel(ProbeRowsArgs a) {
  int cur_len = 0;
  char* out = probe_slot(a, reinterpret_cast<char*>(a.out), &cur_len);
  if (out == nullptr) return;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= a.rows) return;
  const T* x = reinterpret_cast<const T*>(a.x) + (size_t)warp * a.H;
  T* y = reinterpret_cast<T*>(out) + (size_t)(warp / a.q_len) * a.out_b + (size_t)(warp % a.q_len) * a.H;
  if (a.ln_w == nullptr) {
    for (int i = lane; i < a.H; i += 32) __stcs(y + i, x[i]);
    return;
  }
  float s = 0.f;
  for (int i = lane; i < a.H; i += 32) s += DT<T>::to_f(x[i]);
  const float mean = warp_sum(s) / (float)a.H;
  float v = 0.f;
  for (int i = lane; i < a.H; i += 32) { const float d = DT<T>::to_f(x[i]) - mean; v = fmaf(d, d, v); }
  const float rstd = rsqrtf(warp_sum(v) / (float)a.H + a.eps);
  for (int i = lane; i < a.H; i += 32)
    __stcs(y + i, DT<T>::from_f((DT<T>::to_f(x[i]) - mean) * rstd * a.ln_w[i] + a.ln_b[i]));
}

template <typename T, int QT>
static int launch_probs_t(const AttnProbeArgs& a, cudaStream_t st) {
  const size_t smem = (size_t)QT * (HD + a.kv_cap) * sizeof(float);
  PTTS_REQUIRE(smem <= 200 * 1024, "attention_probs: %d keys need %zu B of shared memory (> 200 KB)", a.kv_cap, smem);
  static bool attr = false;
  if (!attr) {
    PTTS_CHECK_CUDA(cudaFuncSetAttribute(attention_probs_kernel<T, QT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  attention_probs_kernel<T, QT><<<dim3((a.q_len + QT - 1) / QT, a.nh, a.B), QT * 32, smem, st>>>(a);
  PTTS_CHECK_CUDA(cudaGetLastError());
  return PTTS_OK;
}

int launch_attention_probs(const AttnProbeArgs& a, int dtype, cudaStream_t st) {
  PTTS_REQUIRE(a.B > 0 && a.nh > 0 && a.nkv > 0 && a.nh % a.nkv == 0 && a.q_len > 0 && a.kv_cap > 0, "attention_probs: bad shape");
  // 8 query rows per CTA wherever there are that many (the key rows are read once per tile), else one
  if (a.q_len >= 8)
    return dtype == PTTS_BF16 ? launch_probs_t<bf16, 8>(a, st) : launch_probs_t<float, 8>(a, st);
  return dtype == PTTS_BF16 ? launch_probs_t<bf16, 1>(a, st) : launch_probs_t<float, 1>(a, st);
}

// One CTA per batch row, one warp per alignment head of this layer (warp w takes the layer's entries w, w + nw, ...).  A head's
// scores are attention_probs_kernel's (the same q load, RoPE, scale, fp32 dot products in the same order, rounded to the model
// dtype), over the key_len transcript keys only; the softmax over those keys alone is the eager weights restricted to them and
// renormalized, before any rounding.  Each warp sums its heads' distributions; the CTA adds the warps in order and scales by
// `weight`.  Cost per row: (heads of the layer) x key_len K rows, independent of the cache length.
template <typename T>
__global__ void __launch_bounds__(256) alignment_probe_kernel(AlignProbeArgs a) {
  extern __shared__ __align__(16) float sma[];
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x, P = a.key_len;
  if (a.ctrl->active == 0) return;
  const int cl = a.ctrl->cur_len;
  const int row = cl - 1 - a.n0 - a.first_row;
  if (row < 0 || row >= a.n_rows) return;
  float* qs = sma + (size_t)warp * (HD + 2 * P);   // [64] the head's scaled, rotated query
  float* sc = qs + HD;                             // [P] its rounded scores (-inf: masked key)
  float* acc = sc + P;                             // [P] this warp's sum of distributions
  for (int p = lane; p < P; p += 32) acc[p] = 0.f;
  const int pos = a.prefix + cl - 1;
  const int kvb = b / a.kv_b_div;
  const int* km = a.key_mask ? a.key_mask + (size_t)kvb * a.mask_ld : nullptr;
  const T* rope_cos = reinterpret_cast<const T*>(a.rope_cos);
  const T* rope_sin = reinterpret_cast<const T*>(a.rope_sin);
  int k = 0;   // index of the entry among this layer's
  for (int e = 0; e < a.n_heads; e++) {
    if (a.heads[2 * e] != a.layer) continue;
    if (k++ % nw != warp) continue;
    const int h = a.heads[2 * e + 1];
    const T* src = reinterpret_cast<const T*>(a.q) + (size_t)b * a.ldq + a.q_col0 + (size_t)h * HD;
    for (int d = lane; d < HD; d += 32) {
      float x = DT<T>::to_f(src[d]);
      if (a.rope) {
        const float xp = DT<T>::to_f(src[d < HD / 2 ? d + HD / 2 : d - HD / 2]);
        x = rope_elem<T>(x, xp, d, rope_cos + (size_t)pos * HD, rope_sin + (size_t)pos * HD);
      }
      qs[d] = DT<T>::rnd(x * a.scale);
    }
    __syncwarp();
    const T* kc = reinterpret_cast<const T*>(a.kcache) + (size_t)kvb * a.kv_b_stride + (size_t)(h / (a.nh / a.nkv)) * a.kv_h_stride;
    float m = -INFINITY;
    for (int p = lane; p < P; p += 32) {
      const int t = a.key0 + p;
      float s = -INFINITY;
      if (km == nullptr || km[t] != 0) {
        const T* krow = kc + (size_t)t * HD;
        float dot = 0.f;
#pragma unroll
        for (int c = 0; c < HD / 8; c++) {
          float kv[8];
          load8(krow + kv_swz(t, 8 * c), kv);
#pragma unroll
          for (int i = 0; i < 8; i++) dot = fmaf(qs[8 * c + i], kv[i], dot);
        }
        s = DT<T>::rnd(dot);
      }
      sc[p] = s;
      m = fmaxf(m, s);
    }
    m = warp_max(m);
    if (m != -INFINITY) {   // every transcript key masked: the head adds nothing
      float l = 0.f;
      for (int p = lane; p < P; p += 32) l += expf(sc[p] - m);
      l = warp_sum(l);
      for (int p = lane; p < P; p += 32) acc[p] += expf(sc[p] - m) / l;
    }
    __syncwarp();
  }
  __syncthreads();
  float* out = a.out + ((size_t)row * a.B + b) * P;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    float v = 0.f;
    for (int w = 0; w < nw; w++) v += sma[(size_t)w * (HD + 2 * P) + HD + P + p];
    v *= a.weight;
    out[p] = a.accumulate ? out[p] + v : v;
  }
}

int launch_alignment_probe(const AlignProbeArgs& a, int dtype, cudaStream_t st) {
  PTTS_REQUIRE(a.B > 0 && a.nh > 0 && a.nkv > 0 && a.nh % a.nkv == 0 && a.key_len > 0 && a.layer_heads > 0 && a.ctrl != nullptr,
               "alignment_probe: bad shape");
  const int nw = a.layer_heads < 8 ? a.layer_heads : 8;
  const size_t smem = (size_t)nw * (HD + 2 * a.key_len) * sizeof(float);
  PTTS_REQUIRE(smem <= 200 * 1024, "alignment_probe: %d transcript keys need %zu B of shared memory (> 200 KB)", a.key_len, smem);
  static bool attr[2] = {false, false};
  if (!attr[dtype == PTTS_BF16]) {
    if (dtype == PTTS_BF16)
      PTTS_CHECK_CUDA(cudaFuncSetAttribute(alignment_probe_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    else
      PTTS_CHECK_CUDA(cudaFuncSetAttribute(alignment_probe_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr[dtype == PTTS_BF16] = true;
  }
  if (dtype == PTTS_BF16) alignment_probe_kernel<bf16><<<a.B, nw * 32, smem, st>>>(a);
  else alignment_probe_kernel<float><<<a.B, nw * 32, smem, st>>>(a);
  PTTS_CHECK_CUDA(cudaGetLastError());
  return PTTS_OK;
}

int launch_probe_rows(const ProbeRowsArgs& a, int dtype, cudaStream_t st) {
  const int blocks = (a.rows * 32 + 255) / 256;
  if (dtype == PTTS_BF16) probe_rows_kernel<bf16><<<blocks, 256, 0, st>>>(a);
  else probe_rows_kernel<float><<<blocks, 256, 0, st>>>(a);
  PTTS_CHECK_CUDA(cudaGetLastError());
  return PTTS_OK;
}

}  // namespace ptts
