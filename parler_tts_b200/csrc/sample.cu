// sample.cu -- logits -> next token, entirely on the device, plus the integer ops around it.
//
// One CTA per row (B*K rows; sample_core.cuh).  Replaces, per decode step:
//   MinNewTokensLengthLogitsProcessor, ParlerTTSLogitsProcessor (logits_processors.py:44-53, stateful:
//   quirk Q11), Temperature/TopK/TopP warpers, softmax + multinomial / argmax, finished-row padding,
//   torch.cat of the history, EosTokenCriteria + MaxLengthCriteria, `unfinished.max()==0` (a host sync
//   per step in the reference) -- i.e. one iteration of transformers' GenerationMixin._sample -- and
//   apply_delay_pattern_mask on the next input (modeling_parler_tts.py:2909, :205-211).
// The step index lives in the device control block so a captured CUDA graph replays unchanged.
// RNG: Philox4x32-10 keyed by the user seed, counter = (row, column): results do not depend on how
// the batch is sharded over GPUs (SURVEY 8e).  torch.multinomial's stream cannot be reproduced
// bit-for-bit (SURVEY hard part 2); sampling parity is distribution-level, greedy is exact.
#include "common.cuh"
#include "kernels.h"
#include "sample_core.cuh"

namespace ptts {

template <int ITEMS, bool EXT, bool RAGGED>
__device__ __forceinline__ void sample_kernel_body(const SampleArgs& p, const int64_t* __restrict__ forced, const ptts_sampling_ext& x,
                                                   const SampleOut& o, const ptts_logits_ext& lx) {
  pdl_launch_dependents();
  pdl_wait();
  if (p.ctrl->active == 0) return;
  const int row = blockIdx.x;           // one CTA per (utterance, codebook) row
  const int cur_len = p.ctrl->cur_len;  // the new token becomes column `cur_len`
  const ptts_gen_params g = *p.gen;
  sample_rows_cta<ITEMS, 1, EXT, RAGGED>(p, g, forced, row, 0, row + 1, cur_len, x, o, lx);
  // last block advances the control block
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int ticket = atomicAdd(&p.ctrl->done_blocks, 1);
    if (ticket == (int)gridDim.x - 1) {
      __threadfence();
      const int n = atomicAdd(&p.ctrl->n_unfinished, 0);
      p.ctrl->cur_len = cur_len + 1;
      p.ctrl->active = (n > 0) ? 1 : 0;
      p.ctrl->steps_run += 1;
      p.ctrl->n_unfinished = 0;
      p.ctrl->done_blocks = 0;
      __threadfence();
    }
  }
}

template <int ITEMS, bool RAGGED>
__global__ void __launch_bounds__(SMP_THREADS) sample_kernel(SampleArgs p, const int64_t* __restrict__ forced) {
  sample_kernel_body<ITEMS, false, RAGGED>(p, forced, ptts_sampling_ext{}, SampleOut{}, ptts_logits_ext{});
}

// the ptts_sampling_ext and ptts_logits_ext stages and the per-step outputs (sample_core.cuh, EXT = true); the knobs, the table
// pointers and the output window come by value, so a captured graph holds them
template <int ITEMS, bool EXT, bool RAGGED>
__global__ void __launch_bounds__(SMP_THREADS) sample_kernel(SampleArgs p, const int64_t* __restrict__ forced, ptts_sampling_ext x,
                                                             SampleOut o, ptts_logits_ext lx) {
  sample_kernel_body<ITEMS, EXT, RAGGED>(p, forced, x, o, lx);
}

int launch_sample(const SampleArgs& a, const int64_t* forced, cudaStream_t st, bool pdl, const ptts_sampling_ext* ext,
                  const SampleOut* out, const ptts_logits_ext* lext) {
  const int BK = a.B * a.K;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(BK);
  cfg.blockDim = dim3(SMP_THREADS);
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  const int items = (a.V + SMP_THREADS - 1) / SMP_THREADS;
  PTTS_REQUIRE(items <= 9, "sample: vocab_size %d > 2304 not supported", a.V);
  PTTS_REQUIRE((out == nullptr && lext == nullptr) || ext != nullptr, "sample: the per-step outputs and the ptts_logits_ext stages need the EXT sampler");
  const bool rg = a.shift != nullptr;
  if (ext != nullptr) {
    const SampleOut o = out ? *out : SampleOut{};
    const ptts_logits_ext lx = lext ? *lext : kLogitsExtOff;
    auto fn = items <= 1 ? (rg ? sample_kernel<1, true, true> : sample_kernel<1, true, false>)
            : items <= 5 ? (rg ? sample_kernel<5, true, true> : sample_kernel<5, true, false>)
                         : (rg ? sample_kernel<9, true, true> : sample_kernel<9, true, false>);
    PTTS_CHECK_CUDA(cudaLaunchKernelEx(&cfg, fn, a, forced, *ext, o, lx));
    return PTTS_OK;
  }
  auto fn = items <= 1 ? (rg ? sample_kernel<1, true> : sample_kernel<1, false>)
          : items <= 5 ? (rg ? sample_kernel<5, true> : sample_kernel<5, false>)
                       : (rg ? sample_kernel<9, true> : sample_kernel<9, false>);
  PTTS_CHECK_CUDA(cudaLaunchKernelEx(&cfg, fn, a, forced));
  return PTTS_OK;
}

// ptts_op_sample_phase: the step kernels' sampling phase (sample_all_rows_cta, passes of up to three rows per CTA) over a grid of
// n_ctas CTAs, on the session's logits.  cur_len stays where it is; the last CTA clears the counters the rows add to.
template <int ITEMS, bool RAGGED>
__global__ void __launch_bounds__(SMP_THREADS) sample_phase_kernel(SampleArgs p) {
  if (p.ctrl->active == 0) return;
  const int cur_len = p.ctrl->cur_len;
  const ptts_gen_params g = *p.gen;
  sample_all_rows_cta<ITEMS, RAGGED>(p, g, (int)blockIdx.x, (int)gridDim.x, p.B * p.K, cur_len);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0 && atomicAdd(&p.ctrl->done_blocks, 1) == (int)gridDim.x - 1) {
    p.ctrl->n_unfinished = 0;
    p.ctrl->done_blocks = 0;
    __threadfence();
  }
}

int launch_sample_phase(const SampleArgs& a, int n_ctas, cudaStream_t st) {
  const int items = (a.V + SMP_THREADS - 1) / SMP_THREADS;
  PTTS_REQUIRE(items <= 9, "sample: vocab_size %d > 2304 not supported", a.V);
  PTTS_REQUIRE(n_ctas >= 1, "op_sample_phase: n_ctas must be positive, got %d", n_ctas);
  const bool rg = a.shift != nullptr;
  auto fn = items <= 1 ? (rg ? sample_phase_kernel<1, true> : sample_phase_kernel<1, false>)
          : items <= 5 ? (rg ? sample_phase_kernel<5, true> : sample_phase_kernel<5, false>)
                       : (rg ? sample_phase_kernel<9, true> : sample_phase_kernel<9, false>);
  fn<<<n_ctas, SMP_THREADS, 0, st>>>(a);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// build_delay_pattern_mask (modeling_parler_tts.py:214-276), cell c of row `row` (codebook k) for the BOS-led ids [B*K][ld], of
// which the first seq columns are the row's input: the id shifted by k, BOS over the lower triangle, PAD over the upper one (:261);
// -1 = free (predicted).  No pattern below 2K-1 columns.
__device__ __forceinline__ int64_t delay_pattern_cell(const int64_t* ids, int row, int ld, int seq, int k, int K, int64_t bos, int64_t pad,
                                                      int L, int c) {
  if (L < 2 * K - 1) return -1;
  const bool bos_pat = c <= k;
  const bool eos_pat = (c - k) >= (L - K + 1);
  const int64_t shifted = (c >= k && c < seq + k) ? ids[(size_t)row * ld + (c - k)] : -1;
  return ((!bos_pat && !eos_pat) ? shifted : 0) + (bos_pat ? bos : 0) + (eos_pat ? pad : 0);
}

// ids == nullptr: the BOS column.  Otherwise the history starts with the delayed input: the first n0 columns of the pattern (:3523;
// where the pattern is free -- max_length < 2K-1 -- the ids themselves), the K-1 cells after it are kept for the sampler's next-input
// override, and eos_seen records the first EOS inside the input (ParlerTTSLogitsProcessor counts the whole history, :46).
// lens != nullptr (ragged): row b does all of this with its own n0_b = lens[b] columns and its own limit L - (n0 - n0_b), exactly
// as the row alone would; its history columns [n0_b, n0) get PAD (the prefill embeds them, and the decode steps overwrite their
// K/V before any query reaches them), and shift[b] = n0 - n0_b.
__global__ void generate_begin_kernel(SampleArgs p, const int64_t* __restrict__ ids, int n0, int L, const int* __restrict__ lens) {
  const int BK = p.B * p.K;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    p.ctrl->cur_len = n0; p.ctrl->active = 1; p.ctrl->n_unfinished = 0; p.ctrl->done_blocks = 0; p.ctrl->steps_run = 0;
    p.ctrl->launch_gen = 0;
    for (int j = 0; j < 32; j++) p.ctrl->bar[j] = 0;
  }
  if (i < BK) {
    if (ids == nullptr) {
      p.raw_ids[(size_t)i * p.raw_ld] = p.bos;
      p.cur_ids[i] = p.bos;
      p.eos_seen[i] = 0;
    } else {
      const int k = i % p.K;
      const int nb = lens != nullptr ? lens[i / p.K] : n0;   // this row's input columns
      const int Lb = L - (n0 - nb);
      int64_t v = 0;
      int es = 0;
      for (int c = 0; c < nb; c++) {
        const int64_t m = delay_pattern_cell(ids, i, n0, nb, k, p.K, p.bos, p.pad, Lb, c);
        v = (m == -1) ? ids[(size_t)i * n0 + c] : m;
        p.raw_ids[(size_t)i * p.raw_ld + c] = v;
        if (v == p.eos && es == 0) es = c + 1;
      }
      for (int c = nb; c < n0; c++) p.raw_ids[(size_t)i * p.raw_ld + c] = p.pad;
      p.cur_ids[i] = (int)v;
      p.eos_seen[i] = es;
      if (p.prefix_cells != nullptr)
        for (int c = 0; c < p.K - 1; c++)
          p.prefix_cells[(size_t)i * (p.K - 1) + c] = delay_pattern_cell(ids, i, n0, nb, k, p.K, p.bos, p.pad, Lb, nb + c);
    }
    p.unfinished[i] = 1;
  }
  if (i < p.B) {
    p.first_unf[i] = i * p.K; p.first_unf[p.B + i] = i * p.K;
    if (lens != nullptr) p.shift[i] = n0 - lens[i];
  }
}
int launch_generate_begin(const SampleArgs& a, const int64_t* ids, int n0, int max_length, const int* lens, cudaStream_t st) {
  const int n = a.B * a.K;
  generate_begin_kernel<<<(n + 127) / 128, 128, 0, st>>>(a, ids, ids == nullptr ? 1 : n0, max_length, lens);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// ---- stand-alone integer operators --------------------------------------------------------------
// build_delay_pattern_mask (modeling_parler_tts.py:214-276): pattern_mask only (bit-exact int64).
__global__ void delay_build_kernel(const int64_t* ids, int BK, int seq, int K, int64_t bos, int64_t pad, int L, int64_t* mask) {
  const int row = blockIdx.x;
  const int k = row % K;
  for (int c = threadIdx.x; c < L; c += blockDim.x) mask[(size_t)row * L + c] = delay_pattern_cell(ids, row, seq, seq, k, K, bos, pad, L, c);
}
int launch_delay_build(const int64_t* ids, int BK, int seq, int K, int64_t bos, int64_t pad, int L, int64_t* mask, cudaStream_t st) {
  delay_build_kernel<<<BK, 128, 0, st>>>(ids, BK, seq, K, bos, pad, L, mask);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}
__global__ void delay_apply_kernel(const int64_t* ids, int seq, int64_t ld_ids, const int64_t* mask, int64_t ld_mask, int64_t* out) {
  const int row = blockIdx.x;
  for (int c = threadIdx.x; c < seq; c += blockDim.x) {
    const int64_t m = mask[(size_t)row * ld_mask + c];
    out[(size_t)row * seq + c] = (m == -1) ? ids[(size_t)row * ld_ids + c] : m;
  }
}
int launch_delay_apply(const int64_t* ids, int BK, int seq, int64_t ld_ids, const int64_t* mask, int64_t ld_mask, int64_t* out, cudaStream_t st) {
  delay_apply_kernel<<<BK, 128, 0, st>>>(ids, seq, ld_ids, mask, ld_mask, out);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// ParlerTTSLogitsProcessor.__call__ on a full history (the HF-loop entry point), one CTA per batch row.
__global__ void logits_processor_kernel(const int64_t* ids, int seq, int64_t ld_ids, float* scores, int V, int64_t eos, int K, int64_t* first_unf) {
  __shared__ int cnt[32];
  const int b = blockIdx.x;
  if (threadIdx.x < 32) cnt[threadIdx.x] = 0;
  __syncthreads();
  for (int k = 0; k < K; k++) {
    int c = 0;
    for (int t = threadIdx.x; t < seq; t += blockDim.x) c += ids[(size_t)(b * K + k) * ld_ids + t] == eos;
    if (c) atomicAdd(&cnt[k], c);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t fu = first_unf[b];
    const int kk = (int)(fu - (int64_t)b * K);
    if (kk >= 0 && kk < K && cnt[kk] > 0 && fu < (int64_t)b * K + K - 1) fu++;
    first_unf[b] = fu;
    for (int k = 0; k < K; k++)
      if ((int64_t)b * K + k > fu) scores[(size_t)(b * K + k) * V + eos] = -INFINITY;
  }
}
int launch_logits_processor(const int64_t* ids, int BK, int seq, int64_t ld_ids, float* scores, int V, int64_t eos, int K, int64_t* first_unf, cudaStream_t st) {
  PTTS_REQUIRE(K <= 32 && BK % K == 0, "logits_processor: bad num_codebooks %d for %d rows", K, BK);
  PTTS_REQUIRE(eos >= 0 && eos < V, "`eos_token_id` has to be in [0, vocab), got %lld", (long long)eos);
  logits_processor_kernel<<<BK / K, 128, 0, st>>>(ids, seq, ld_ids, scores, V, eos, K, first_unf);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

}  // namespace ptts
