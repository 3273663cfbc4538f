// score.cu -- teacher-forced scoring (ptts_score): the K lm heads over every label position and the cross-entropy of the
// reference's loss (modeling_parler_tts.py:1922-1974), without materialising the logits.
//
// Why: scoring B utterances of T frames needs B*T*K rows of V logits -- at Mini, B = 32 and T = 430 that is 539 MB of fp32
// the reference writes and reads back.  What the loss needs per (row, codebook) is log-sum-exp and one logit, so the fused
// kernel keeps a running max / sum of exp per row in registers while it sweeps the codebook's V columns tile by tile, and
// writes one fp32 NLL per (row, codebook).  It is the prefill GEMM's pipeline (wgmma.cuh) over a row-major copy of the
// LayerNorm-folded heads (ptts_lm_heads_rowmajor_pack), with the epilogue of the heads GEMM: the folded LayerNorm
// (ln_stats.cuh) and rounding to bf16, so its logits are the unfused path's up to the accumulation order.
//
// The unfused route (fp32 sessions, or when the caller wants the logits) runs the decoder's own heads GEMM one frame at a time
// (B rows) into the workspace logits and then score_rows_kernel below over those fp32 rows.
#include <cfloat>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace ptts {
namespace score {

using wg::K_STAGE;
using wg::M_TILE;
constexpr int NT = 128;  // vocabulary columns per n-tile (V = 1088 is 8.5 tiles: the last one is zero-filled and masked)

// Label of row r = b*T + t, codebook k, as the loss counts it: -1 where the reference's mask drops it (:1935-1946: a BOS label
// becomes -100; a cell counts iff its decoder input id != eos and its label != -100).
__device__ __forceinline__ int target_of(const ScoreArgs& a, int r, int k) {
  const int b = r / a.T, t = r - b * a.T;
  const int64_t lab = a.labels[(int64_t)r * a.K + k];
  const int64_t dec = a.dec_ids[((int64_t)b * a.K + k) * a.T + t];
  return (lab == -100 || lab == a.bos || dec == a.eos) ? -1 : (int)lab;
}

// Label row r = b*T + t of the decoder's output x [B][P + T][H] -> xs [B*T][H] contiguous (the fused kernel's TMA operand),
// plus its LayerNorm (mean, rstd) like row_stats_kernel (gemm_tc.cu).  One warp per row.
__global__ void gather_label_rows_kernel(const bf16* __restrict__ x, int P, int T, int H, int M, float eps, bf16* __restrict__ xs,
                                         float* __restrict__ stats) {
  const int r = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= M) return;
  const int b = r / T, t = r - b * T;
  const bf16* src = x + ((size_t)b * (P + T) + P + t) * H;
  bf16* dst = xs + (size_t)r * H;
  float s = 0.f;
  for (int k = lane; k < H; k += 32) { const bf16 v = src[k]; dst[k] = v; s += __bfloat162float(v); }
  const float mean = warp_sum(s) / (float)H;
  float q = 0.f;
  for (int k = lane; k < H; k += 32) { const float d = __bfloat162float(src[k]) - mean; q = fmaf(d, d, q); }
  const float var = warp_sum(q) / (float)H;
  if (lane == 0) { stats[2 * r] = mean; stats[2 * r + 1] = rsqrtf(var + eps); }
}

// One CTA: rows m0 .. m0+127 of xs against codebook blockIdx.y's V heads rows, n-tile by n-tile.  Per (row, codebook):
// nll = logsumexp(logits) - logits[label], in the log2 domain (exp2 of pre-scaled values) inside the sweep.  One CTA per SM:
// the 64 accumulators plus the per-row state need more than the ~96 registers two CTAs would leave (ptxas spills there).
__global__ void __launch_bounds__(wg::THREADS, 1)
ce_fused_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, const ScoreArgs a,
                const float* __restrict__ stats) {
  extern __shared__ unsigned char smem_raw[];
  const wg::Pipe pipe = wg::pipe_setup<NT>(smem_raw);
  const int V = a.V, cb = blockIdx.y, m0 = blockIdx.x * M_TILE;
  float* cvec = reinterpret_cast<float*>(pipe.extra);  // [2][V]: c1 | c2 of this codebook
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
  }
  for (int c = threadIdx.x; c < V; c += blockDim.x) { cvec[c] = a.c1[(int64_t)cb * V + c]; cvec[V + c] = a.c2[(int64_t)cb * V + c]; }
  __syncthreads();

  const int n_k = a.H / K_STAGE, n_tiles = (V + NT - 1) / NT, n_iter = n_tiles * n_k;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == wg::PRODUCER_WARP) {  // the K loops of all n-tiles as one stream of stages
    if (lane == 0) {
      for (int g = 0; g < n_iter; g++) {
        const int s = g % wg::STAGES, use = g / wg::STAGES, j = g / n_k, kk = g - j * n_k;
        if (use > 0) wg::mbar_wait(&pipe.empty[s], (use - 1) & 1);
        unsigned char* a_dst = pipe.stages + (size_t)s * wg::STAGE_BYTES<NT>;
        mbar_expect_tx(&pipe.full[s], (uint32_t)(wg::A_BYTES + NT * K_STAGE * 2));
        wg::tma_load_2d(a_dst, &map_x, kk * K_STAGE, m0, &pipe.full[s]);
        wg::tma_load_3d(a_dst + wg::A_BYTES, &map_w, kk * K_STAGE, j * NT, cb, &pipe.full[s]);
      }
    }
    return;
  }

  // this thread's two rows (h = 0, 1): statistics, label, and the running (max, sum of exp2) of its columns
  const int rbase = m0 + 64 * (warp >> 2);
  float mean[2], rstd[2], run_m[2], run_s[2], lab_v[2];
  int tgt[2];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int r = rbase + wg::frag_row(2 * h);
    const bool ok = r < a.M;
    mean[h] = ok ? stats[2 * r] : 0.f;
    rstd[h] = ok ? stats[2 * r + 1] : 0.f;
    tgt[h] = ok ? target_of(a, r, cb) : -1;
    run_m[h] = -FLT_MAX; run_s[h] = 0.f; lab_v[h] = 0.f;
  }
  const float LOG2E = 1.4426950408889634f;

  float acc[NT / 2];
  const uint32_t a_row0 = (uint32_t)(warp >> 2) * 64 * 128;
  for (int j = 0; j < n_tiles; j++) {
    for (int kk = 0; kk < n_k; kk++) {
      const int g = j * n_k + kk, s = g % wg::STAGES;
      wg::mbar_wait(&pipe.full[s], (g / wg::STAGES) & 1);
      const uint32_t a_addr = smem_u32(pipe.stages + (size_t)s * wg::STAGE_BYTES<NT>);
      const uint64_t da = wg::desc_sw128(a_addr + a_row0), db = wg::desc_sw128(a_addr + wg::A_BYTES);
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int k = 0; k < K_STAGE / 16; k++) wg::mma<NT>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kk > 0 || k > 0) ? 1 : 0);
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
      if (g > 0 && lane == 0) wg::mbar_arrive(&pipe.empty[(g - 1) % wg::STAGES]);
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    // epilogue of n-tile j: logits (folded LayerNorm, rounded to bf16 like the heads GEMM), then the online log-sum-exp; the
    // logit of register i is recomputed for the sum rather than kept
#pragma unroll
    for (int h = 0; h < 2; h++) {
      float tmax = -FLT_MAX;
#pragma unroll
      for (int i0 = 0; i0 < NT / 2; i0 += 4)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int i = i0 + 2 * h + e, c = j * NT + wg::frag_col(i);
          if (c < V) {
            const float v = DT<bf16>::rnd(rstd[h] * (acc[i] - mean[h] * cvec[c]) + cvec[V + c]);
            if (c == tgt[h]) lab_v[h] = v;
            tmax = fmaxf(tmax, v);
          }
        }
      const float nm = fmaxf(run_m[h], tmax * LOG2E);
      float sum = 0.f;
#pragma unroll
      for (int i0 = 0; i0 < NT / 2; i0 += 4)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int i = i0 + 2 * h + e, c = j * NT + wg::frag_col(i);
          if (c < V) sum += exp2f(DT<bf16>::rnd(rstd[h] * (acc[i] - mean[h] * cvec[c]) + cvec[V + c]) * LOG2E - nm);
        }
      run_s[h] = run_s[h] * exp2f(run_m[h] - nm) + sum;
      run_m[h] = nm;
    }
  }
  // the four threads of a quad hold the same rows: combine their (max, sum) and the one label logit
#pragma unroll
  for (int h = 0; h < 2; h++) {
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, run_m[h], o), os = __shfl_xor_sync(0xffffffffu, run_s[h], o);
      const float nm = fmaxf(run_m[h], om);
      run_s[h] = run_s[h] * exp2f(run_m[h] - nm) + os * exp2f(om - nm);
      run_m[h] = nm;
      lab_v[h] += __shfl_xor_sync(0xffffffffu, lab_v[h], o);
    }
    const int r = rbase + wg::frag_row(2 * h);
    if ((lane & 3) == 0 && r < a.M) {
      const float lse = (run_m[h] + log2f(run_s[h])) * 0.6931471805599453f;
      a.token_nll[(int64_t)r * a.K + cb] = tgt[h] >= 0 ? lse - lab_v[h] : 0.f;
    }
  }
}

// Unfused route, frame t: logits [B*K][V] f32 (the heads GEMM's output for the B rows of frame t) -> token_nll[b][t][k]
// (when labels are given) and a copy into logits_out [B*K][T][V] (when requested).  One block per (b, k) row.
__global__ void score_rows_kernel(const float* __restrict__ logits, int t, const ScoreArgs a, float* __restrict__ logits_out) {
  const int row = blockIdx.x, b = row / a.K, k = row - b * a.K, V = a.V;
  const float* lr = logits + (size_t)row * V;
  if (logits_out != nullptr) {
    float* o = logits_out + ((size_t)row * a.T + t) * V;
    for (int c = threadIdx.x; c < V; c += blockDim.x) o[c] = lr[c];
  }
  if (a.labels == nullptr) return;
  __shared__ float red[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float m = -FLT_MAX;
  for (int c = threadIdx.x; c < V; c += blockDim.x) m = fmaxf(m, lr[c]);
  m = warp_max(m);
  if (lane == 0) red[w] = m;
  __syncthreads();
  m = red[0];
  for (int i = 1; i < nw; i++) m = fmaxf(m, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int c = threadIdx.x; c < V; c += blockDim.x) s += expf(lr[c] - m);
  s = warp_sum(s);
  if (lane == 0) red[w] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    s = 0.f;
    for (int i = 0; i < nw; i++) s += red[i];
    const int r = b * a.T + t, tg = target_of(a, r, k);
    a.token_nll[(int64_t)r * a.K + k] = tg >= 0 ? (m + logf(s)) - lr[tg] : 0.f;
  }
}

// Per-codebook sum of token_nll and count of counted cells, over rows in a fixed order (one block per codebook, a fixed
// thread-to-row map and a fixed tree): the same inputs give the same bits on every run.
__global__ void ce_reduce_kernel(const ScoreArgs a, float* __restrict__ out) {
  constexpr int NTH = 256;
  __shared__ double ssum[NTH];
  __shared__ int scnt[NTH];
  const int k = blockIdx.x;
  double s = 0.0;
  int n = 0;
  for (int r = threadIdx.x; r < a.M; r += NTH) {
    if (target_of(a, r, k) < 0) continue;
    s += (double)a.token_nll[(int64_t)r * a.K + k];
    n++;
  }
  ssum[threadIdx.x] = s; scnt[threadIdx.x] = n;
  __syncthreads();
  for (int w = NTH / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) { ssum[threadIdx.x] += ssum[threadIdx.x + w]; scnt[threadIdx.x] += scnt[threadIdx.x + w]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { out[2 * k] = (float)ssum[0]; out[2 * k + 1] = (float)scnt[0]; }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// bf16 tensor of `rank` dims (dims[0] contiguous), box {64, box_rows, 1}, 128-byte swizzle, zero fill outside the tensor
static int make_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, uint32_t box_rows) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
    if (!fn) return fail(PTTS_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");
  }
  cuuint64_t strides[2] = {dims[0] * 2, dims[0] * dims[1] * 2};
  cuuint32_t box[3] = {(cuuint32_t)K_STAGE, box_rows, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(PTTS_ECUDA, "cuTensorMapEncodeTiled failed (%d) for the scoring operands", (int)r);
  return PTTS_OK;
}

}  // namespace score

bool score_fused_supported(int H, int V) { return H % score::K_STAGE == 0 && V % 8 == 0 && V <= 8192; }

int launch_score_fused(const ScoreArgs& a, const void* x, int P, float eps, void* xs_scratch, float* stats_scratch,
                       const void* heads_rm, cudaStream_t st) {
  using namespace score;
  PTTS_REQUIRE(score_fused_supported(a.H, a.V), "score: the fused kernel needs hidden_size %% 64 == 0 and vocab_size <= 8192");
  const int warps_per_block = 8;
  gather_label_rows_kernel<<<(a.M + warps_per_block - 1) / warps_per_block, warps_per_block * 32, 0, st>>>(
      (const bf16*)x, P, a.T, a.H, a.M, eps, (bf16*)xs_scratch, stats_scratch);
  PTTS_LAUNCH_CHECK();
  CUtensorMap mx, mw;
  const cuuint64_t dx[2] = {(cuuint64_t)a.H, (cuuint64_t)a.M};
  const cuuint64_t dw[3] = {(cuuint64_t)a.H, (cuuint64_t)a.V, (cuuint64_t)a.K};  // [K][V][H]: each codebook's tail is zero-filled
  if (int e = make_map(&mx, xs_scratch, 2, dx, (uint32_t)M_TILE)) return e;
  if (int e = make_map(&mw, heads_rm, 3, dw, (uint32_t)NT)) return e;
  const size_t smem = wg::smem_bytes<NT>(2 * a.V * (int)sizeof(float));
  PTTS_CHECK_CUDA(cudaFuncSetAttribute(ce_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((a.M + M_TILE - 1) / M_TILE, a.K, 1);
  ce_fused_kernel<<<grid, wg::THREADS, smem, st>>>(mx, mw, a, stats_scratch);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

int launch_score_rows(const ScoreArgs& a, const float* logits, int t, float* logits_out, cudaStream_t st) {
  score::score_rows_kernel<<<a.B * a.K, 256, 0, st>>>(logits, t, a, logits_out);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

int launch_score_reduce(const ScoreArgs& a, float* out, cudaStream_t st) {
  score::ce_reduce_kernel<<<a.K, 256, 0, st>>>(a, out);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

}  // namespace ptts
