// gemm.cu -- weight-streaming linear layers of the decoder step.
//
// y[M, N] = epilogue( LN?(x[M, K]) @ W[N, K]^T )       (all decoder nn.Linear are bias-free, Q4)
// Replaces the cuBLAS calls behind q/k/v/out_proj (modeling_parler_tts.py:855, :877-878, :928),
// fc1/fc2 (:1060-1062), the K lm heads (:1920) and the nn.LayerNorm launches in front of them
// (:1020, :1040, :1059, :1632).
//
// Roofline: at decode M = batch (32) so every weight byte is used 2*M flop-times: HBM-bound
// (algorithmic bytes = 2*N*K).  Design for bandwidth, not tensor throughput:
//   * weights are pre-shuffled at load into mma.m16n8k16 B-fragment order: one LDG.128 per lane =
//     one fully-coalesced 512 B request per warp, no shared-memory staging for the big operand;
//   * the 32-row activation tile (64 KB for H=1024) is staged once in shared memory, LayerNorm is
//     applied in place (fp32 statistics, output rounded to the model dtype like torch);
//   * 8 warps split K (interleaved 32-wide slabs -> the CTA streams contiguous 4 KB), partial
//     accumulators are reduced through shared memory in a fixed order (deterministic);
//   * weight prefetch is issued BEFORE griddepcontrol.wait so that under programmatic dependent
//     launch the HBM stream of kernel i+1 overlaps the tail of kernel i.
// The f32 model dtype (config 1, CPU-parity runs) uses a plain SIMT tile kernel.
#include "common.cuh"
#include "kernels.h"
#include "ln_stats.cuh"
#include "ptx.cuh"

namespace ptts {

// ---- bf16 tensor-core path ----------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

constexpr int GEMM_THREADS = 256;
constexpr int GEMM_WARPS = 8;
constexpr int TILE_M = 32;

template <int NT, int PF>
__global__ void __launch_bounds__(GEMM_THREADS) linear_bf16_kernel(LinearArgs p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float ln_stats[64];        // (mean, rstd) per row when LayerNorm is folded in
  __shared__ float ln_part[8 * 32 * 2];  // per-warp partial (S1, S2), ln_stats.cuh
  bf16* xs = reinterpret_cast<bf16*>(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Kc = p.Kc, lds = Kc + 8;
  const int kt_per_chunk = Kc >> 5;
  const int n_chunks = p.K / Kc;
  const int KT = p.K >> 5;  // 32-wide k slabs in the whole matrix
  const int nt0 = blockIdx.x * NT;
  const int m0 = blockIdx.y * TILE_M;
  const uint4* __restrict__ W = reinterpret_cast<const uint4*>(p.W);

  // per-warp slab schedule: slab index (within a chunk) = warp + 8*i
  const int per_chunk = (kt_per_chunk > warp) ? (kt_per_chunk - warp + GEMM_WARPS - 1) / GEMM_WARPS : 0;

  uint4 wr[PF][NT];
  auto load_w = [&](uint4 (&dst)[NT], int c, int i) {
    const int ktg = c * kt_per_chunk + warp + GEMM_WARPS * i;  // global 32-wide slab index
#pragma unroll
    for (int j = 0; j < NT; j++) dst[j] = ldg_stream(W + ((size_t)(nt0 + j) * KT + ktg) * 32 + lane);
  };
  // Weights do not depend on the previous kernel: start the HBM stream before the grid dependency.
#pragma unroll
  for (int s = 0; s < PF; s++)
    if (s < per_chunk) load_w(wr[s], 0, s);

  pdl_launch_dependents();
  pdl_wait();
  if (p.ctrl != nullptr && p.ctrl->active == 0) return;

  float acc[2][NT][4];
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int j = 0; j < NT; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[a][j][e] = 0.f;

  RowStatFrag rst;
  row_stat_zero(rst);
  const bf16* __restrict__ X = reinterpret_cast<const bf16*>(p.X);
  for (int c = 0; c < n_chunks; c++) {
    if (c > 0) {
      // this warp is done with the previous chunk's slots: refill them before the block-wide sync
#pragma unroll
      for (int s = 0; s < PF; s++)
        if (s < per_chunk) load_w(wr[s], c, s);
      __syncthreads();  // previous chunk fully consumed by every warp
    }
    // stage x[m0:m0+32, c*Kc:(c+1)*Kc] (rows >= M are zero)
    const int vec_per_row = Kc >> 3;
    for (int v = threadIdx.x; v < TILE_M * vec_per_row; v += GEMM_THREADS) {
      const int r = v / vec_per_row, cv = v - r * vec_per_row;
      uint4 val = make_uint4(0, 0, 0, 0);
      if (m0 + r < p.M) val = *reinterpret_cast<const uint4*>(X + (size_t)(m0 + r) * p.ldx + (size_t)c * Kc + cv * 8);
      *reinterpret_cast<uint4*>(xs + r * lds + cv * 8) = val;
    }
    __syncthreads();
    if (p.c1 != nullptr) row_stat_pass(rst, xs, lds, kt_per_chunk, warp, lane);  // tensor-core row sums (ln_stats.cuh)
    const int lrow = (lane & 7) + ((lane >> 3) & 1) * 8;
    const int lcol = (lane >> 4) * 8;
    for (int i0 = 0; i0 < per_chunk; i0 += PF) {
#pragma unroll
      for (int s = 0; s < PF; s++) {
        const int i = i0 + s;
        if (i < per_chunk) {
          const int kt = warp + GEMM_WARPS * i;  // slab inside the staged chunk
          uint32_t a[2][2][4];
#pragma unroll
          for (int mt = 0; mt < 2; mt++)
#pragma unroll
            for (int j = 0; j < 2; j++) ldmatrix_x4(a[mt][j], xs + (mt * 16 + lrow) * lds + kt * 32 + j * 16 + lcol);
#pragma unroll
          for (int j = 0; j < NT; j++) {
            const uint4 w = wr[s][j];
#pragma unroll
            for (int mt = 0; mt < 2; mt++) {
              mma_bf16_16816(acc[mt][j], a[mt][0], w.x, w.y);
              mma_bf16_16816(acc[mt][j], a[mt][1], w.z, w.w);
            }
          }
          if (i + PF < per_chunk) load_w(wr[s], c, i + PF);
        }
      }
    }
  }
  if (p.c1 != nullptr) row_stat_store(rst, ln_part, warp, lane);
  __syncthreads();
  if (p.c1 != nullptr) row_stat_finalize(ln_part, p.K, p.M - m0, p.eps, ln_stats);  // published by the barrier before the epilogue
  // cross-warp K reduction in fixed order, then epilogue
  float* red = reinterpret_cast<float*>(smem_raw);  // [8][32][8*NT]
  constexpr int FB = 8 * NT;
  {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
      for (int j = 0; j < NT; j++) {
        float* base = red + ((size_t)warp * TILE_M + mt * 16 + g) * FB + j * 8 + 2 * t;
        base[0] = acc[mt][j][0];
        base[1] = acc[mt][j][1];
        base[8 * FB] = acc[mt][j][2];
        base[8 * FB + 1] = acc[mt][j][3];
      }
  }
  __syncthreads();
  const int n0 = nt0 * 8;
  for (int o = threadIdx.x; o < TILE_M * FB; o += GEMM_THREADS) {
    const int r = o / FB, cidx = o - r * FB;
    if (m0 + r >= p.M) continue;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < GEMM_WARPS; w++) v += red[((size_t)w * TILE_M + r) * FB + cidx];
    if (p.c1 != nullptr) v = ln_stats[2 * r + 1] * (v - ln_stats[2 * r] * p.c1[n0 + cidx]) + p.c2[n0 + cidx];
    v = DT<bf16>::rnd(v);  // nn.Linear output is rounded to the model dtype
    const size_t yo = (size_t)(m0 + r) * p.ldy + n0 + cidx;
    if (p.epi == EPI_ACT) {
      v = apply_act(v, p.act);
    } else if (p.epi == EPI_RESIDUAL) {
      v = DT<bf16>::to_f(reinterpret_cast<const bf16*>(p.R)[(size_t)(m0 + r) * p.ldr + n0 + cidx]) + v;
    }
    if (p.epi == EPI_F32) reinterpret_cast<float*>(p.Y)[yo] = v;
    else reinterpret_cast<bf16*>(p.Y)[yo] = __float2bfloat16_rn(v);
  }
}

// ---- f32 SIMT path (parity mode) ----------------------------------------------------------------
// 32 rows x 32 features per CTA, 256 threads, 4 outputs per thread, K in slabs of 32.
__global__ void __launch_bounds__(256) linear_f32_kernel(LinearArgs p) {
  __shared__ float xs[32][33];
  __shared__ float ws[32][33];
  __shared__ float mean_s[32], rstd_s[32];
  pdl_launch_dependents();
  pdl_wait();
  if (p.ctrl != nullptr && p.ctrl->active == 0) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  const float* __restrict__ X = reinterpret_cast<const float*>(p.X);
  const float* __restrict__ W = reinterpret_cast<const float*>(p.W);
  if (p.ln_w != nullptr) {
    for (int r = ty; r < 32; r += 8) {
      float mean = 0.f, rstd = 0.f;
      if (m0 + r < p.M) {
        const float* row = X + (size_t)(m0 + r) * p.ldx;
        float s = 0.f;
        for (int c = tx; c < p.K; c += 32) s += row[c];
        mean = warp_sum(s) / (float)p.K;
        float q = 0.f;
        for (int c = tx; c < p.K; c += 32) { float d = row[c] - mean; q += d * d; }
        rstd = rsqrtf(warp_sum(q) / (float)p.K + p.eps);
      }
      if (tx == 0) { mean_s[r] = mean; rstd_s[r] = rstd; }
    }
    __syncthreads();
  }
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k0 = 0; k0 < p.K; k0 += 32) {
    for (int r = ty; r < 32; r += 8) {
      float xv = 0.f;
      if (m0 + r < p.M) {
        xv = X[(size_t)(m0 + r) * p.ldx + k0 + tx];
        if (p.ln_w != nullptr) xv = (xv - mean_s[r]) * rstd_s[r] * p.ln_w[k0 + tx] + p.ln_b[k0 + tx];
      }
      xs[r][tx] = xv;
      ws[r][tx] = (n0 + r < p.N) ? W[(size_t)(n0 + r) * p.K + k0 + tx] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < 32; kk++) {
      const float wv = ws[tx][kk];
#pragma unroll
      for (int i = 0; i < 4; i++) acc[i] = fmaf(xs[ty + 8 * i][kk], wv, acc[i]);
    }
    __syncthreads();
  }
  const int n = n0 + tx;
  if (n >= p.N) return;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int m = m0 + ty + 8 * i;
    if (m >= p.M) continue;
    float v = acc[i];
    if (p.epi == EPI_ACT) v = apply_act(v, p.act);
    else if (p.epi == EPI_RESIDUAL) v = reinterpret_cast<const float*>(p.R)[(size_t)m * p.ldr + n] + v;
    reinterpret_cast<float*>(p.Y)[(size_t)m * p.ldy + n] = v;
  }
}

// ---- host launch --------------------------------------------------------------------------------
template <int NT, int PF>
static int launch_bf16(const LinearArgs& a, cudaStream_t st, bool pdl) {
  const int lds = a.Kc + 8;
  size_t smem = (size_t)TILE_M * lds * sizeof(bf16);
  size_t red = (size_t)GEMM_WARPS * TILE_M * 8 * NT * sizeof(float);
  if (red > smem) smem = red;
  static bool attr_done = false;  // per instantiation
  if (!attr_done) {
    PTTS_CHECK_CUDA(cudaFuncSetAttribute(linear_bf16_kernel<NT, PF>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attr_done = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(a.N / (8 * NT), (a.M + TILE_M - 1) / TILE_M);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  PTTS_CHECK_CUDA(cudaLaunchKernelEx(&cfg, linear_bf16_kernel<NT, PF>, a));
  return PTTS_OK;
}

int launch_linear(const LinearArgs& a_in, int dtype, cudaStream_t st, bool pdl, int sm_count) {
  LinearArgs a = a_in;
  PTTS_REQUIRE(a.M > 0 && a.N > 0 && a.K > 0, "linear: empty problem M=%d N=%d K=%d", a.M, a.N, a.K);
  if (dtype == PTTS_F32) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((a.N + 31) / 32, (a.M + 31) / 32);
    cfg.blockDim = dim3(256);
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    PTTS_CHECK_CUDA(cudaLaunchKernelEx(&cfg, linear_f32_kernel, a));
    return PTTS_OK;
  }
  PTTS_REQUIRE(a.K % 32 == 0 && a.N % 8 == 0, "linear: need K%%32==0 and N%%8==0 (K=%d N=%d)", a.K, a.N);
  if (a.Kc <= 0) {
    // activation tile width: whole row when LayerNorm is fused, else the largest slab <= 1536 dividing K
    a.Kc = a.K;
    if (a.ln_w == nullptr && a.K > 1536) {
      for (int d = 2; d <= 64; d++)
        if (a.K % d == 0 && (a.K / d) % 32 == 0 && a.K / d <= 1536) { a.Kc = a.K / d; break; }
    }
  }
  PTTS_REQUIRE(a.Kc <= 2048 && a.K % a.Kc == 0 && a.Kc % 32 == 0, "linear: bad K tile %d for K=%d", a.Kc, a.K);
  // n-tiles per CTA: the largest tile that still gives ~one CTA per SM (132 on an H100) for this matrix; fewer,
  // fatter CTAs mean fewer copies of the 32-row activation tile pulled through the L2->SM crossbar.  (Restated by ntile_pick in tests/test_linear_reference.py, which asserts the decode shapes reach every variant: keep the two in step.)
  const int ntiles = a.N / 8;
  const int cand[6] = {8, 6, 4, 3, 2, 1};
  const int want = ntiles < (sm_count * 85) / 100 ? ntiles : (sm_count * 85) / 100;
  int best = 1;
  for (int i = 0; i < 6; i++) {
    if (ntiles % cand[i]) continue;
    if (ntiles / cand[i] >= want) { best = cand[i]; break; }
  }
  switch (best) {
    case 1: return launch_bf16<1, 4>(a, st, pdl);
    case 2: return launch_bf16<2, 4>(a, st, pdl);
    case 3: return launch_bf16<3, 4>(a, st, pdl);
    case 4: return launch_bf16<4, 4>(a, st, pdl);
    case 6: return launch_bf16<6, 2>(a, st, pdl);
    default: return launch_bf16<8, 2>(a, st, pdl);
  }
}

// ---- weight repacking (load time) ---------------------------------------------------------------
template <typename S>
__global__ void pack_matrix_bf16_kernel(const S* __restrict__ src, int64_t rows, int64_t cols, int row_off, int K, bf16* __restrict__ dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int64_t r = i / cols, k = i - r * cols;
  const int64_t n = r + row_off;
  const int64_t nt = n >> 3, g = n & 7, kt = k >> 5, kk = k & 31;
  const int j = (int)(kk >> 4), c = (int)(kk & 15), half = c >> 3, t = (c & 7) >> 1, e = c & 1;
  const int lane = (int)g * 4 + t, reg = j * 2 + half;
  const int64_t off = ((nt * (K >> 5) + kt) * 32 + lane) * 8 + reg * 2 + e;
  float v;
  if constexpr (sizeof(S) == 2) v = __bfloat162float(src[i]); else v = src[i];
  dst[off] = __float2bfloat16_rn(v);
}
template <typename S, typename D>
__global__ void pack_plain_kernel(const S* __restrict__ src, int64_t n, D* __restrict__ dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v;
  if constexpr (sizeof(S) == 2) v = __bfloat162float(src[i]); else v = src[i];
  if constexpr (sizeof(D) == 2) dst[i] = __float2bfloat16_rn(v); else dst[i] = v;
}

int pack_matrix(const void* src, int src_dtype, int64_t rows, int64_t cols, int row_off, int K, void* dst, int dst_dtype, cudaStream_t st) {
  const int64_t n = rows * cols;
  const int threads = 256;
  const int blocks = (int)((n + threads - 1) / threads);
  if (dst_dtype == PTTS_BF16) {
    if (src_dtype == PTTS_BF16) pack_matrix_bf16_kernel<bf16><<<blocks, threads, 0, st>>>((const bf16*)src, rows, cols, row_off, K, (bf16*)dst);
    else pack_matrix_bf16_kernel<float><<<blocks, threads, 0, st>>>((const float*)src, rows, cols, row_off, K, (bf16*)dst);
  } else {
    float* d = (float*)dst + (int64_t)row_off * K;
    if (src_dtype == PTTS_BF16) pack_plain_kernel<bf16, float><<<blocks, threads, 0, st>>>((const bf16*)src, n, d);
    else pack_plain_kernel<float, float><<<blocks, threads, 0, st>>>((const float*)src, n, d);
  }
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// W (fragment order, bf16) <- bf16(gamma_k * W_nk);  c1_n = sum_k W'_nk;  c2_n = sum_k beta_k * W_nk   (one block per row n)
__global__ void __launch_bounds__(128) fold_layernorm_kernel(bf16* __restrict__ wp, int K, const float* __restrict__ g, const float* __restrict__ b,
                                                             float* __restrict__ c1, float* __restrict__ c2) {
  __shared__ float sh[8];
  const int n = blockIdx.x;
  const int64_t nt = n >> 3, gq = n & 7;
  float a1 = 0.f, a2 = 0.f;
  for (int k = threadIdx.x; k < K; k += 128) {
    const int64_t kt = k >> 5;
    const int kk = k & 31, j = kk >> 4, c = kk & 15, half = c >> 3, t = (c & 7) >> 1, e = c & 1;
    const int64_t off = ((nt * (K >> 5) + kt) * 32 + (gq * 4 + t)) * 8 + (j * 2 + half) * 2 + e;
    const float w = __bfloat162float(wp[off]);
    a2 = fmaf(b[k], w, a2);
    const bf16 wf = __float2bfloat16_rn(g[k] * w);
    wp[off] = wf;
    a1 += __bfloat162float(wf);
  }
  a1 = warp_sum(a1);
  a2 = warp_sum(a2);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sh[warp] = a1; sh[4 + warp] = a2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    c1[n] = (sh[0] + sh[1]) + (sh[2] + sh[3]);
    c2[n] = (sh[4] + sh[5]) + (sh[6] + sh[7]);
  }
}
int fold_layernorm(void* w_packed, int N, int K, const float* gamma, const float* beta, float* c1, float* c2, cudaStream_t st) {
  fold_layernorm_kernel<<<N, 128, 0, st>>>((bf16*)w_packed, K, gamma, beta, c1, c2);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

int pack_plain(const void* src, int src_dtype, int64_t n, void* dst, int dst_dtype, cudaStream_t st) {
  const int threads = 256;
  const int blocks = (int)((n + threads - 1) / threads);
  if (src_dtype == PTTS_BF16 && dst_dtype == PTTS_BF16) pack_plain_kernel<bf16, bf16><<<blocks, threads, 0, st>>>((const bf16*)src, n, (bf16*)dst);
  else if (src_dtype == PTTS_BF16) pack_plain_kernel<bf16, float><<<blocks, threads, 0, st>>>((const bf16*)src, n, (float*)dst);
  else if (dst_dtype == PTTS_BF16) pack_plain_kernel<float, bf16><<<blocks, threads, 0, st>>>((const float*)src, n, (bf16*)dst);
  else pack_plain_kernel<float, float><<<blocks, threads, 0, st>>>((const float*)src, n, (float*)dst);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

}  // namespace ptts
