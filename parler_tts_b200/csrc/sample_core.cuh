// sample_core.cuh -- one row of logits -> next token (shared by sample_kernel and the fused step kernel).
#pragma once
#include <cfloat>
#include "common.cuh"
#include "kernels.h"

namespace ptts {

__device__ __forceinline__ uint32_t fkey(float f) {  // order-preserving float -> uint
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
  const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
  c[0] = hi1 ^ c[1] ^ k0; c[1] = lo1; c[2] = hi0 ^ c[3] ^ k1; c[3] = lo0;
}
__device__ __forceinline__ float philox_uniform(uint64_t seed, uint32_t row, uint32_t col) {
  uint32_t c[4] = {row, col, 0x5054u, 0x5453u};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; i++) { philox_round(c, k0, k1); k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
  return (float)(c[0] >> 8) * (1.0f / 16777216.0f);  // [0, 1)
}


// Processes up to R rows (row0, row0 + stride, ...; those >= n_rows are skipped) with ONE CTA of SMP_THREADS threads (element i of a
// row lives on thread i % 256, slot i / 256): the bitwise top-k / top-p searches, the softmax sums and the inverse-CDF draw are
// CTA-wide reductions / scans with a fixed order (lanes by butterfly, then warps 0..7), so results are bit-reproducible and identical
// between sample_kernel (R = 1) and the fused step kernels (both run exactly this code; per row the arithmetic does not depend on R).
// The R rows share every CTA barrier: a row is mostly latency (two dependent L2 loads up front, 32 barrier-separated search
// iterations, 10 more for the draw, three dependent global accesses at the end), so three rows per pass take little longer than one
// and the step kernel's 288 rows need one pass instead of three rounds back to back.
// One warp per row would leave 75 % of the fused kernel's warps idle and hold 72 live values per lane.
// Every thread of the CTA must call it (it contains __syncthreads()).
constexpr int SMP_WARPS = 8;
constexpr int SMP_THREADS = SMP_WARPS * 32;

constexpr int SMP_MAX_ROWS = 3;
struct SmpScratch {
  float f[2][SMP_MAX_ROWS][SMP_WARPS];
  int i[2][SMP_MAX_ROWS][SMP_WARPS];
  int z[2][SMP_MAX_ROWS][SMP_WARPS];
};
__device__ __forceinline__ SmpScratch& smp_scratch() {
  __shared__ SmpScratch sc;
  return sc;
}
// EXT: the no_repeat_ngram bans of each row, one bit per id of the largest vocabulary a CTA takes (9 slots of 256)
constexpr int SMP_BAN_WORDS = 9 * SMP_THREADS / 32;
__device__ __forceinline__ uint32_t (&smp_bans())[SMP_MAX_ROWS][SMP_BAN_WORDS] {
  __shared__ uint32_t ban[SMP_MAX_ROWS][SMP_BAN_WORDS];
  return ban;
}
// EXT: the sequence_bias sequences of each row whose prefix matches the history: the id they bias (-1: no match), and their biases
struct SmpSeq {
  int last[SMP_MAX_ROWS][PTTS_SEQ_BIAS_MAX];
  float bias[PTTS_SEQ_BIAS_MAX];
};
__device__ __forceinline__ SmpSeq& smp_seq() {
  __shared__ SmpSeq sq;
  return sq;
}
__device__ __forceinline__ bool bitmap_has(const uint32_t* __restrict__ bits, int i) { return (__ldg(bits + (i >> 5)) >> (i & 31)) & 1u; }

// EXT = true adds the ptts_sampling_ext stages (sample_kernel's second set of instantiations): the n-gram bans join the EOS masks,
// and MinP, Typical, Epsilon and Eta run after top-p on the same arrays, each a fixed-order CTA reduction or a bitwise threshold
// search, so draws stay bit-reproducible.  With every stage off it computes what EXT = false computes.  EXT = true also records
// generate()'s per-step outputs when the step (cur_len - input_len) lies in o's window: the raw row as loaded, and the final
// processed row where p.scores gets it.
// EXT = true also runs the ptts_logits_ext stages (lx; the caller passes the off values of ptts_generate_set_logits_ext when none
// is set, not a zeroed struct).  The masks among them (suppress, begin-suppress) join the single mask pass; while an additive,
// forcing or InfNan stage acts on this step, the pass applies every stage per id in transformers' order instead (they do not
// commute with the masks).  Additions and the decay product use __fadd_rn / __fmul_rn so that no FMA changes their rounding.
// RAGGED = true reads each row's column from p.shift (a ragged continuation); RAGGED = false is the code of a uniform batch, in
// which every row samples column cur_len (the callers pick the instantiation by p.shift != nullptr).
// SLOT = true (with RAGGED and EXT; ptts_generate_set_slots) is slot mode: every row is a request of its own that started from
// the BOS column at its own column 0, so its stop, MinNewTokens and delay pattern count in its column col = cur_len - shift[b]
// (stop and pattern at its own limit max_len[b], not max_length) and its draws use the Philox substream key[b] * K + k.
template <int ITEMS, int R, bool EXT = false, bool RAGGED = false, bool SLOT = false>
__device__ __forceinline__ void sample_rows_cta(const SampleArgs& p, const ptts_gen_params& g, const int64_t* __restrict__ forced,
                                                int row0, int stride, int n_rows, int cur_len, ptts_sampling_ext x = {},
                                                SampleOut o = {}, ptts_logits_ext lx = {}, const int* __restrict__ key = nullptr, const int* __restrict__ max_len = nullptr) {
  static_assert(!SLOT || (RAGGED && EXT), "slot mode runs on the ragged EXT sampler");
  static_assert(R >= 1 && R <= SMP_MAX_ROWS, "rows per pass");
  SmpScratch& sc = smp_scratch();   // one static buffer for every instantiation inlined into a kernel
  float (&s_f)[2][SMP_MAX_ROWS][SMP_WARPS] = sc.f;
  int (&s_i)[2][SMP_MAX_ROWS][SMP_WARPS] = sc.i;
  int (&s_z)[2][SMP_MAX_ROWS][SMP_WARPS] = sc.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int buf = 0;  // reductions alternate between two scratch rows: a warp may enter the next reduction while others still read this one
  auto cta_sum_i = [&](int (&v)[R]) {
#pragma unroll
    for (int r = 0; r < R; r++) {
      const int w = __reduce_add_sync(0xffffffffu, v[r]);
      if (lane == 0) s_i[buf][r][warp] = w;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < R; r++) {
      int a = 0;
#pragma unroll
      for (int w = 0; w < SMP_WARPS; w++) a += s_i[buf][r][w];
      v[r] = a;
    }
    buf ^= 1;
  };
  auto cta_sum_f = [&](float (&v)[R]) {
#pragma unroll
    for (int r = 0; r < R; r++) {
      const float w = warp_sum(v[r]);
      if (lane == 0) s_f[buf][r][warp] = w;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < R; r++) {
      float a = 0.f;
#pragma unroll
      for (int w = 0; w < SMP_WARPS; w++) a += s_f[buf][r][w];
      v[r] = a;
    }
    buf ^= 1;
  };
  auto cta_max_f = [&](float (&v)[R]) {
#pragma unroll
    for (int r = 0; r < R; r++) {
      const float w = warp_max(v[r]);
      if (lane == 0) s_f[buf][r][warp] = w;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < R; r++) {
      float a = s_f[buf][r][0];
#pragma unroll
      for (int w = 1; w < SMP_WARPS; w++) a = fmaxf(a, s_f[buf][r][w]);
      v[r] = a;
    }
    buf ^= 1;
  };

  int row[R];
  bool valid[R];
  int col[R];   // the column row r samples: its own history's (cur_len less the row's shift in a ragged continuation)
  float v[R][ITEMS];
#pragma unroll
  for (int r = 0; r < R; r++) {
    row[r] = row0 + r * stride;
    valid[r] = row[r] < n_rows;
    col[r] = cur_len - ((RAGGED && valid[r]) ? row_shift(p.shift, row[r] / p.K) : 0);
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      const int i = tid + SMP_THREADS * j;
      v[r][j] = (valid[r] && i < p.V) ? __ldcg(p.logits + (size_t)row[r] * p.V + i) : -INFINITY;  // written by other CTAs of this launch: L2, not L1
    }
  }
  // this step's slot of row r in an output buffer of o (nullptr: not recorded); recomputed where used, nothing stays live
  auto out_row = [&](float* base, int r) -> float* {
    const int step = cur_len - (g.input_len > 1 ? g.input_len : 1);
    if (base == nullptr || !valid[r] || step < o.first_step || step - o.first_step >= o.n_steps) return nullptr;
    return base + (int64_t)(step - o.first_step) * o.step_stride + (int64_t)row[r] * p.V;
  };
  if constexpr (EXT) {  // the raw rows, before any processor (streaming stores: the host reads them after the loop)
#pragma unroll
    for (int r = 0; r < R; r++) {
      if (float* dst = out_row(o.logits, r)) {
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
          const int i = tid + SMP_THREADS * j;
          if (i < p.V) __stcs(dst + i, v[r][j]);
        }
      }
    }
  }
  // the tail's inputs (thread r finishes row r): requested now, consumed after the draw
  int t_unf = 0, t_es = 0;
  if (tid < R && row0 + tid * stride < n_rows) { t_unf = p.unfinished[row0 + tid * stride]; t_es = p.eos_seen[row0 + tid * stride]; }
  // NoRepeatNGram over the row's history, columns [0, col): every i in [0, col - n] whose ids[i, i + n - 1) equal the last
  // n - 1 ids bans ids[i + n - 1].  Nothing is banned while col + 1 < n (cur_len is the largest col of the batch).
  const int ngram = EXT ? x.no_repeat_ngram_size : 0;
  const bool bans = EXT && ngram > 0 && cur_len + 1 >= ngram;
  if constexpr (EXT) {
    if (bans) {
      uint32_t (&ban)[SMP_MAX_ROWS][SMP_BAN_WORDS] = smp_bans();
#pragma unroll
      for (int r = 0; r < R; r++)
        for (int w = tid; w < SMP_BAN_WORDS; w += SMP_THREADS) ban[r][w] = 0u;
      __syncthreads();
#pragma unroll
      for (int r = 0; r < R; r++) {
        if (!valid[r] || col[r] + 1 < ngram) continue;
        const int64_t* h = p.raw_ids + (size_t)row[r] * p.raw_ld;
        const int64_t* tail = h + col[r] - ngram + 1;
        for (int i = tid; i <= col[r] - ngram; i += SMP_THREADS) {
          bool match = true;
          for (int q = 0; q < ngram - 1 && match; q++) match = h[i + q] == tail[q];
          const int64_t t = h[i + ngram - 1];
          if (match && t >= 0 && t < p.V) atomicOr(&ban[r][t >> 5], 1u << (t & 31));
        }
      }
      __syncthreads();
    }
  }
  // ptts_logits_ext: which stages act on this column.  ForcedEOS, the decay and MinNewTokens count from the input's end or the
  // limit, which a ragged row has at the same batch column as every other row (its n0 and max_length are the batch's less its
  // shift), so they stay on cur_len; ForcedBOS and begin-suppress test the row's own column.
  const bool seq_bias = EXT && (lx.bias1 != nullptr || lx.n_seq > 0);
  const bool forced_eos = EXT && lx.forced_eos_token_id >= 0 && cur_len == g.max_length - 1;
  const bool decay = EXT && lx.decay != nullptr && cur_len > lx.decay_start;
  bool forced_bos[R], begin_sup[R];
#pragma unroll
  for (int r = 0; r < R; r++) {
    forced_bos[r] = EXT && lx.forced_bos_token_id >= 0 && col[r] == 1;
    // a ragged row continuing from the BOS column alone begins one column later under a forced BOS, as it would alone
    const int sh = cur_len - col[r];
    const int begin = lx.begin_index - sh + ((sh > 0 && g.input_len - sh == 1 && lx.forced_bos_token_id >= 0) ? 1 : 0);
    begin_sup[r] = EXT && lx.begin_suppress != nullptr && col[r] == begin;
  }
  if constexpr (EXT) {
    if (lx.n_seq > 0) {  // one thread per (row, sequence): does the history end with the sequence's first len - 1 ids?
      SmpSeq& sq = smp_seq();
#pragma unroll
      for (int r = 0; r < R; r++) {
        for (int q = tid; q < lx.n_seq; q += SMP_THREADS) {
          const int32_t* e = lx.seq + q * (1 + PTTS_SEQ_BIAS_MAX_LEN);
          const int len = e[0];
          int last = -1;
          if (valid[r] && len >= 2 && len <= PTTS_SEQ_BIAS_MAX_LEN && len <= col[r]) {
            const int64_t* h = p.raw_ids + (size_t)row[r] * p.raw_ld + col[r] - (len - 1);
            bool match = true;
            for (int t = 0; t < len - 1 && match; t++) match = h[t] == e[1 + t];
            if (match) last = e[len];
          }
          sq.last[r][q] = last;
          if (r == 0) sq.bias[q] = lx.seq_bias[q];
        }
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int r = 0; r < R; r++) {
    const int b = row[r] / p.K, k = row[r] - b * p.K;
    bool mask_eos = false;
    // MinNewTokensLength: prompt_length_to_skip = the decoder input's columns (the BOS column, or n0 when continuing); a slot's
    // request has the BOS column only
    if ((SLOT ? col[r] - 1 : cur_len - (g.input_len > 1 ? g.input_len : 1)) < g.min_new_tokens) mask_eos = true;
    const bool mask_min = mask_eos;   // (EXT's ordered pass applies the two EOS masks at their own places)
    bool mask_par = false;
    // ParlerTTSLogitsProcessor (stateful; state double-buffered on the column parity)
    if (valid[r]) {
      const int par = cur_len & 1;
      int fu = p.first_unf[par * p.B + b];
      // eos_seen[r] = 1 + column of row r's first EOS (0 = none).  The reference counts EOS over input_ids, i.e. columns
      // < col (logits_processors.py:46): an EOS written by another CTA during THIS step (column col) must not count,
      // so the test is on the column, not on a flag (rows of one batch item are sampled by different CTAs).
      const int es = __ldcg(p.eos_seen + fu);
      if (es > 0 && es <= col[r] && fu < b * p.K + p.K - 1) fu++;
      if (k == 0 && tid == 0) p.first_unf[(par ^ 1) * p.B + b] = fu;
      if (row[r] > fu) mask_eos = mask_par = true;
    }
    if (seq_bias || forced_bos[r] || forced_eos || decay || (EXT && lx.remove_invalid_values)) {
      // transformers' order: SequenceBias, NoRepeatNGram, MinNewTokens, ForcedBOS, ForcedEOS, InfNan, ExponentialDecay, Suppress,
      // SuppressAtBegin, ParlerTTS (the custom list is merged last); suppress_special (a bench aid) goes with the last mask
      const float mult = decay ? __ldg(lx.decay + cur_len) : 0.f;
#pragma unroll
      for (int j = 0; j < ITEMS; j++) {
        const int i = tid + SMP_THREADS * j;
        if (i >= p.V) continue;   // padding slots stay -inf (InfNan would lift them)
        float y = v[r][j];
        if (seq_bias) {   // bias = (0 + bias1[i]) + each matching sequence ending in i, in table order; then scores + bias
          float bs = lx.bias1 != nullptr ? __fadd_rn(0.f, __ldg(lx.bias1 + i)) : 0.f;
          for (int q = 0; q < lx.n_seq; q++)
            if (smp_seq().last[r][q] == i) bs = __fadd_rn(bs, smp_seq().bias[q]);
          y = __fadd_rn(y, bs);
        }
        if (bans && ((smp_bans()[r][i >> 5] >> (i & 31)) & 1u)) y = -INFINITY;
        if (mask_min && i == p.eos) y = -INFINITY;
        if (forced_bos[r]) y = (i == lx.forced_bos_token_id) ? 0.f : -INFINITY;
        if (forced_eos) y = (i == lx.forced_eos_token_id) ? 0.f : -INFINITY;
        if (lx.remove_invalid_values) y = (y != y) ? 0.f : (y == INFINITY ? FLT_MAX : (y == -INFINITY ? -FLT_MAX : y));
        if (decay) y = __fadd_rn(y, i == p.eos ? __fmul_rn(fabsf(y), mult) : 0.f);   // scores + penalties (0 off EOS)
        if (lx.suppress != nullptr && bitmap_has(lx.suppress, i)) y = -INFINITY;
        if (begin_sup[r] && bitmap_has(lx.begin_suppress, i)) y = -INFINITY;
        if (mask_par && i == p.eos) y = -INFINITY;
        if (g.suppress_special && i >= g.codebook_size) y = -INFINITY;
        v[r][j] = y;
      }
      continue;
    }
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      const int i = tid + SMP_THREADS * j;
      if (mask_eos && i == p.eos) v[r][j] = -INFINITY;
      if (g.suppress_special && i >= g.codebook_size) v[r][j] = -INFINITY;
      if constexpr (EXT) {
        if (bans && ((smp_bans()[r][i >> 5] >> (i & 31)) & 1u)) v[r][j] = -INFINITY;
        if (i < p.V && lx.suppress != nullptr && bitmap_has(lx.suppress, i)) v[r][j] = -INFINITY;
        if (i < p.V && begin_sup[r] && bitmap_has(lx.begin_suppress, i)) v[r][j] = -INFINITY;
      }
    }
  }
  int tok[R];
#pragma unroll
  for (int r = 0; r < R; r++) tok[r] = 0;
  const bool renorm = EXT && lx.renormalize_logits;
  float n_max[R], n_log[R];  // LogitNormalization: the final row's max and log of its softmax sum
  if (g.do_sample) {
    if (g.temperature != 1.0f) {
#pragma unroll
      for (int r = 0; r < R; r++)
#pragma unroll
        for (int j = 0; j < ITEMS; j++) v[r][j] = v[r][j] / g.temperature;
    }
    if (g.top_k > 0) {
      const int kk = g.top_k < p.V ? g.top_k : p.V;
      uint32_t key[R][ITEMS];
      uint32_t th[R];
#pragma unroll
      for (int r = 0; r < R; r++) {
        th[r] = 0;
#pragma unroll
        for (int j = 0; j < ITEMS; j++) key[r][j] = (tid + SMP_THREADS * j < p.V) ? fkey(v[r][j]) : 0u;   // 0 < every candidate
      }
      for (int bit = 31; bit >= 0; bit--) {  // bitwise binary search of the k-th largest key
        int cnt[R];
#pragma unroll
        for (int r = 0; r < R; r++) {
          const uint32_t cand = th[r] | (1u << bit);
          cnt[r] = 0;
#pragma unroll
          for (int j = 0; j < ITEMS; j++) cnt[r] += (key[r][j] >= cand) ? 1 : 0;
        }
        cta_sum_i(cnt);
#pragma unroll
        for (int r = 0; r < R; r++)
          if (cnt[r] >= kk) th[r] |= (1u << bit);
      }
#pragma unroll
      for (int r = 0; r < R; r++)
#pragma unroll
        for (int j = 0; j < ITEMS; j++)
          if (fkey(v[r][j]) < th[r]) v[r][j] = -INFINITY;  // scores < kth largest
    }
    float m[R];
#pragma unroll
    for (int r = 0; r < R; r++) {
      m[r] = -INFINITY;
#pragma unroll
      for (int j = 0; j < ITEMS; j++) m[r] = fmaxf(m[r], v[r][j]);
    }
    cta_max_f(m);
    float e[R][ITEMS];
    float s[R];
#pragma unroll
    for (int r = 0; r < R; r++) {
      s[r] = 0.f;
#pragma unroll
      for (int j = 0; j < ITEMS; j++) { e[r][j] = expf(v[r][j] - m[r]); s[r] += e[r][j]; }
    }
    cta_sum_f(s);
    if (g.top_p < 1.0f) {
      // remove tokens whose ascending cumulative probability is <= 1 - top_p (the max is always kept)
      uint32_t th[R];
#pragma unroll
      for (int r = 0; r < R; r++) th[r] = 0;
      for (int bit = 31; bit >= 0; bit--) {
        float c[R];
#pragma unroll
        for (int r = 0; r < R; r++) {
          const uint32_t cand = th[r] | (1u << bit);
          c[r] = 0.f;
#pragma unroll
          for (int j = 0; j < ITEMS; j++) c[r] += (fkey(v[r][j]) <= cand) ? e[r][j] : 0.f;
        }
        cta_sum_f(c);
#pragma unroll
        for (int r = 0; r < R; r++)
          if (c[r] <= (1.0f - g.top_p) * s[r]) th[r] |= (1u << bit);
      }
#pragma unroll
      for (int r = 0; r < R; r++) {
        const uint32_t kmax = fkey(m[r]);
        s[r] = 0.f;
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
          const uint32_t key = fkey(v[r][j]);
          if (key <= th[r] && key != kmax) { v[r][j] = -INFINITY; e[r][j] = 0.f; }
          s[r] += e[r][j];
        }
      }
      cta_sum_f(s);
    }
    if constexpr (EXT) {
      // The warpers after top-p (transformers' order: MinP, Typical, Epsilon, Eta).  Each sees the softmax of the scores the
      // previous one left: p_j = e_j / s with e_j = exp(v_j - m).  The max is never removed, so m stays the max.
      auto drop_where = [&](auto&& remove) {
#pragma unroll
        for (int r = 0; r < R; r++) {
          const float inv = 1.0f / s[r];
          s[r] = 0.f;
#pragma unroll
          for (int j = 0; j < ITEMS; j++) {
            if (remove(r, j, inv)) { v[r][j] = -INFINITY; e[r][j] = 0.f; }
            s[r] += e[r][j];
          }
        }
        cta_sum_f(s);
      };
      // entropy -sum p log p of the current scores, with log p = v - m - log s (log_softmax); removed ids add nothing
      auto entropy = [&](float (&ent)[R], float (&lse)[R]) {
#pragma unroll
        for (int r = 0; r < R; r++) {
          lse[r] = m[r] + logf(s[r]);
          ent[r] = 0.f;
#pragma unroll
          for (int j = 0; j < ITEMS; j++)
            if (v[r][j] > -INFINITY) { const float lp = v[r][j] - lse[r]; ent[r] += lp * expf(lp); }
        }
        cta_sum_f(ent);
#pragma unroll
        for (int r = 0; r < R; r++) ent[r] = -ent[r];
      };
      if (x.min_p > 0.f)  // p < min_p * p_max; p_max = 1 / s
        drop_where([&](int r, int j, float inv) { return e[r][j] * inv < x.min_p * inv; });
      if (x.typical_p < 1.0f) {
        // shifted_j = |-log p_j - H|.  Sorted ascending, the first position whose cumulative p reaches the mass gives the
        // threshold T; ids with shifted > T go.  T is found as the key after the largest key th with mass(shifted <= th) < typical_p.
        float ent[R], lse[R];
        entropy(ent, lse);
        uint32_t key[R][ITEMS], th[R];
#pragma unroll
        for (int r = 0; r < R; r++) {
          th[r] = 0;
#pragma unroll
          for (int j = 0; j < ITEMS; j++) key[r][j] = fkey(v[r][j] > -INFINITY ? fabsf(lse[r] - v[r][j] - ent[r]) : INFINITY);
        }
        for (int bit = 31; bit >= 0; bit--) {
          float c[R];
#pragma unroll
          for (int r = 0; r < R; r++) {
            const uint32_t cand = th[r] | (1u << bit);
            c[r] = 0.f;
#pragma unroll
            for (int j = 0; j < ITEMS; j++) c[r] += (key[r][j] <= cand) ? e[r][j] : 0.f;
          }
          cta_sum_f(c);
#pragma unroll
          for (int r = 0; r < R; r++)
            if (c[r] < x.typical_p * s[r]) th[r] |= (1u << bit);
        }
        // th = 0xffffffff: the mass is never reached (rounding), the threshold is the largest shifted value and nothing goes
        drop_where([&](int r, int j, float) { return th[r] != 0xffffffffu && key[r][j] > th[r] + 1u; });
      }
      if (x.epsilon_cutoff > 0.f)
        drop_where([&](int r, int j, float inv) { return e[r][j] * inv < x.epsilon_cutoff && v[r][j] < m[r]; });
      if (x.eta_cutoff > 0.f) {
        float ent[R], lse[R];
        entropy(ent, lse);
        drop_where([&](int r, int j, float inv) {
          return e[r][j] * inv < fminf(x.eta_cutoff, sqrtf(x.eta_cutoff) * expf(-ent[r])) && v[r][j] < m[r];
        });
      }
    }
    // inverse-CDF draw in index order: CTA-wide inclusive scan per slot j (elements 256 j .. 256 j + 255)
    float target[R], carry[R];
    int found[R], last_nz[R];
#pragma unroll
    for (int r = 0; r < R; r++) {
      const uint32_t stream = !SLOT ? (uint32_t)(row[r] + g.row_base) : valid[r] ? (uint32_t)(key[row[r] / p.K] * p.K + row[r] % p.K) : 0u;
      target[r] = philox_uniform(g.seed, stream, (uint32_t)col[r]) * s[r];
      carry[r] = 0.f; found[r] = -1; last_nz[r] = -1;
    }
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      float x[R];
#pragma unroll
      for (int r = 0; r < R; r++) {
        x[r] = e[r][j];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const float y = __shfl_up_sync(0xffffffffu, x[r], o);
          if (lane >= o) x[r] += y;
        }
        if (lane == 31) s_f[buf][r][warp] = x[r];  // this warp's total
      }
      __syncthreads();
      float tot[R];
#pragma unroll
      for (int r = 0; r < R; r++) {
        float base = carry[r];
        tot[r] = carry[r];
#pragma unroll
        for (int w = 0; w < SMP_WARPS; w++) {
          const float tw = s_f[buf][r][w];
          if (w < warp) base += tw;
          tot[r] += tw;
        }
        const float cum = base + x[r];
        const unsigned hit = __ballot_sync(0xffffffffu, cum > target[r] && e[r][j] > 0.f);
        const unsigned nz = __ballot_sync(0xffffffffu, e[r][j] > 0.f);
        if (lane == 0) {
          s_i[buf][r][warp] = hit ? SMP_THREADS * j + 32 * warp + (__ffs(hit) - 1) : 0x7fffffff;
          s_z[buf][r][warp] = nz ? SMP_THREADS * j + 32 * warp + (31 - __clz(nz)) : -1;
        }
      }
      __syncthreads();
#pragma unroll
      for (int r = 0; r < R; r++) {
        int first = 0x7fffffff, lastz = -1;
#pragma unroll
        for (int w = 0; w < SMP_WARPS; w++) { first = min(first, s_i[buf][r][w]); lastz = max(lastz, s_z[buf][r][w]); }
        if (found[r] < 0 && first != 0x7fffffff) found[r] = first;
        if (lastz >= 0) last_nz[r] = lastz;
        carry[r] = tot[r];
      }
      buf ^= 1;
    }
#pragma unroll
    for (int r = 0; r < R; r++) tok[r] = found[r] >= 0 ? found[r] : last_nz[r];
    if constexpr (EXT) {  // every id removed (the bans can do that): token 0, as greedy's argmax gives
#pragma unroll
      for (int r = 0; r < R; r++) {
        if (tok[r] < 0) tok[r] = 0;
        n_max[r] = m[r];          // the warpers never remove the max
        n_log[r] = logf(s[r]);
      }
    }
  } else {
    // argmax, smallest index on ties
#pragma unroll
    for (int r = 0; r < R; r++) {
      float m = -INFINITY;
      int mi = 0x7fffffff;
#pragma unroll
      for (int j = 0; j < ITEMS; j++) {
        const int i = tid + SMP_THREADS * j;
        if (i < p.V && (v[r][j] > m || (v[r][j] == m && i < mi))) { m = v[r][j]; mi = i; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, o);
        const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
        if (om > m || (om == m && oi < mi)) { m = om; mi = oi; }
      }
      if (lane == 0) { s_f[buf][r][warp] = m; s_i[buf][r][warp] = mi; }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < R; r++) {
      float m = s_f[buf][r][0];
      int mi = s_i[buf][r][0];
#pragma unroll
      for (int w = 1; w < SMP_WARPS; w++) {
        const float om = s_f[buf][r][w];
        const int oi = s_i[buf][r][w];
        if (om > m || (om == m && oi < mi)) { m = om; mi = oi; }
      }
      tok[r] = mi;
    }
    buf ^= 1;
    if (renorm) {  // greedy: the argmax above is taken before the normalization
#pragma unroll
      for (int r = 0; r < R; r++) {
        n_max[r] = -INFINITY;
#pragma unroll
        for (int j = 0; j < ITEMS; j++) n_max[r] = fmaxf(n_max[r], v[r][j]);
      }
      cta_max_f(n_max);
#pragma unroll
      for (int r = 0; r < R; r++) {
        n_log[r] = 0.f;
#pragma unroll
        for (int j = 0; j < ITEMS; j++) n_log[r] += expf(v[r][j] - n_max[r]);
      }
      cta_sum_f(n_log);
#pragma unroll
      for (int r = 0; r < R; r++) n_log[r] = logf(n_log[r]);
    }
  }
  if (renorm) {  // log_softmax = (x - max) - log(sum exp(x - max))
#pragma unroll
    for (int r = 0; r < R; r++)
#pragma unroll
      for (int j = 0; j < ITEMS; j++) v[r][j] = (v[r][j] - n_max[r]) - n_log[r];
  }
#pragma unroll
  for (int r = 0; r < R; r++) {
    if (!valid[r]) continue;
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      const int i = tid + SMP_THREADS * j;
      if (i < p.V) p.scores[(size_t)row[r] * p.V + i] = v[r][j];
    }
    if constexpr (EXT) {
      if (float* dst = out_row(o.scores, r)) {
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
          const int i = tid + SMP_THREADS * j;
          if (i < p.V) __stcs(dst + i, v[r][j]);
        }
      }
    }
  }
  // thread r finishes row r (the rows are independent: each owns its entries of every array below)
  int my_tok = 0, my_row = 0, my_col = 0;
  bool my_valid = false;
#pragma unroll
  for (int r = 0; r < R; r++)
    if (tid == r) { my_tok = tok[r]; my_row = row[r]; my_valid = valid[r]; my_col = col[r]; }
  if (tid < R && my_valid) {
    const int b = my_row / p.K, k = my_row - b * p.K;
    int t = my_tok;
    if (forced != nullptr) t = (int)forced[my_row];
    if (!t_unf) t = p.pad;  // next_tokens * unfinished + pad * (1 - unfinished)
    p.raw_ids[(size_t)my_row * p.raw_ld + my_col] = t;
    if (t == p.eos && t_es == 0) p.eos_seen[my_row] = my_col + 1;
    // the row's own limit max_length - shift is reached at the batch's max_length; a slot's limit is max_len[b] in its column
    const int new_len = (SLOT ? my_col : cur_len) + 1;
    const int done = (t == p.eos) || (new_len >= (SLOT ? max_len[b] : g.max_length));
    const int still_unfinished = t_unf && !done;
    p.unfinished[my_row] = still_unfinished;
    // delay-pattern override of the NEXT model input (column `my_col`), build_delay_pattern_mask :252-261, with the row's own
    // limit Lb and input length nb
    const int sh = cur_len - my_col;
    const int Lb = SLOT ? max_len[b] : g.max_length - sh, nb = SLOT ? 1 : g.input_len - sh;
    int nxt = t;
    if (Lb >= 2 * p.K - 1) {
      const bool is_bos = my_col <= k;
      const bool is_pad = (my_col - k) >= (Lb - p.K + 1);
      if (is_bos || is_pad) nxt = (is_bos ? p.bos : 0) + (is_pad ? p.pad : 0);
      // continuing from n0 input columns: codebook k's prefix ids reach up to column n0-1+k, past the delayed input (:246-248)
      else if (nb > 1 && my_col - nb < k) nxt = (int)p.prefix_cells[(size_t)my_row * (p.K - 1) + (my_col - nb)];
    }
    p.cur_ids[my_row] = nxt;
    if (still_unfinished) atomicAdd(&p.ctrl->n_unfinished, 1);
  }
  __syncthreads();  // the scratch rows may be reused by the next pass of this CTA
}

template <int ITEMS>
__device__ __forceinline__ void sample_row_cta(const SampleArgs& p, const ptts_gen_params& g, const int64_t* __restrict__ forced,
                                               int row, int cur_len) {
  sample_rows_cta<ITEMS, 1>(p, g, forced, row, 0, row + 1, cur_len);
}

// all rows of the token over the CTAs of a fused step kernel: passes of up to three rows per CTA
template <int ITEMS, bool RAGGED = false>
__device__ __forceinline__ void sample_all_rows_cta(const SampleArgs& p, const ptts_gen_params& g, int cta, int n_ctas, int n_rows, int cur_len) {
  if (n_rows <= n_ctas) {
    if (cta < n_rows) sample_rows_cta<ITEMS, 1, false, RAGGED>(p, g, nullptr, cta, n_ctas, n_rows, cur_len);
  } else {
    for (int row0 = cta; row0 < n_rows; row0 += 3 * n_ctas) sample_rows_cta<ITEMS, 3, false, RAGGED>(p, g, nullptr, row0, n_ctas, n_rows, cur_len);
  }
}

}  // namespace ptts
