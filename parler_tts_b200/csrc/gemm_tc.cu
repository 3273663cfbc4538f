// gemm_tc.cu -- the prefill linear layers as Hopper wgmma GEMMs (bf16 model dtype; what linear_tc_supported rejects, and fp32, run
// the mma.sync kernel of gemm.cu; tests/test_linear_reference.py checks both against float64 at every tile edge).
//
// Why: at prefill the decoder's linear layers see M = B*(P+1) (prompt) or B*S (encoder K/V projection) rows, ~1000-2000 for
// the bench workload: 6.6 GFLOP per matrix, tensor-bound.  The decode GEMM (gemm.cu: 32-row tiles, mma.sync, weights re-read
// from L2 for every 32 rows) is the wrong shape for them.  A 128-row x up-to-128-feature tile with TMA-fed 128-byte-swizzled
// operands is the same machinery as the DAC convolutions (dac_tc.cu: a k=1 convolution over channels-last activations IS
// x W^T), so this kernel is that pipeline (wgmma.cuh) with the nn.Linear epilogues of the reference
// (modeling_parler_tts.py:1020-1062): optional folded LayerNorm (y = rstd*(acc - mean*c1) + c2, ln_stats.cuh), rounding to
// bf16, GELU, residual add.  Feature tiles stop at 128 columns: 64 fp32 accumulators per thread keep two CTAs per SM, and the
// narrower tiles give these small-M matrices enough CTAs to cover the 132 SMs.
#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace ptts {
namespace gtc {

using wg::M_TILE;
using wg::K_STAGE;

struct Args {
  int M, N, K;
  const float* stats;  // [M][2] (mean, rstd) per row, or nullptr (no folded LayerNorm)
  const float* c1;     // [N] folded-LayerNorm vectors (with stats)
  const float* c2;
  int epi, act;
  const bf16* R;       // residual [M][N] (EPI_RESIDUAL)
  bf16* Y;             // [M][N]
};

// One CTA: Y[m0:m0+128, n0:n0+NT] = epilogue( X[m0:m0+128, :] W[n0:n0+NT, :]^T ), X and W row-major bf16 (K contiguous).
template <int NT>
__global__ void __launch_bounds__(wg::THREADS, 2)
linear_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, const Args p) {
  extern __shared__ unsigned char smem_raw[];
  const wg::Pipe pipe = wg::pipe_setup<NT>(smem_raw);
  float* cvec = reinterpret_cast<float*>(pipe.extra);  // [2][NT]: c1 | c2
  const int m0 = blockIdx.x * M_TILE, n0 = blockIdx.y * NT;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
  }
  if (p.stats != nullptr)
    for (int c = threadIdx.x; c < NT; c += blockDim.x) { cvec[c] = p.c1[n0 + c]; cvec[NT + c] = p.c2[n0 + c]; }
  __syncthreads();

  float acc[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; i++) acc[i] = 0.f;
  auto load = [&](int it, unsigned char* a_dst, unsigned char* b_dst, uint64_t* bar) {
    wg::tma_load_2d(a_dst, &map_x, it * K_STAGE, m0, bar);
    wg::tma_load_2d(b_dst, &map_w, it * K_STAGE, n0, bar);
  };
  wg::mainloop<NT>(pipe, p.K / K_STAGE, load, acc);
  if ((threadIdx.x >> 5) == wg::PRODUCER_WARP) return;

  // ===== epilogue: each register pair is two adjacent columns of one row =====
  const int mrow = m0 + 64 * (threadIdx.x >> 7);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int m = mrow + wg::frag_row(2 * h);
    if (m >= p.M) continue;
    float mean = 0.f, rstd = 1.f;
    if (p.stats != nullptr) { mean = p.stats[2 * m]; rstd = p.stats[2 * m + 1]; }
    const size_t orow = (size_t)m * p.N + n0;
#pragma unroll
    for (int j = 0; j < NT / 8; j++) {
      const int i = 4 * j + 2 * h, c = wg::frag_col(i);
      float a = acc[i], b = acc[i + 1];
      if (p.stats != nullptr) {
        a = rstd * (a - mean * cvec[c]) + cvec[NT + c];
        b = rstd * (b - mean * cvec[c + 1]) + cvec[NT + c + 1];
      }
      a = DT<bf16>::rnd(a); b = DT<bf16>::rnd(b);  // nn.Linear output is rounded to the model dtype
      if (p.epi == EPI_ACT) { a = apply_act(a, p.act); b = apply_act(b, p.act); }
      else if (p.epi == EPI_RESIDUAL) {
        const float2 rr = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.R + orow + c));
        a = rr.x + a; b = rr.y + b;
      }
      *reinterpret_cast<__nv_bfloat162*>(p.Y + orow + c) = __floats2bfloat162_rn(a, b);
    }
  }
}

// (mean, rstd) per row of a bf16 [M][K] matrix: fp32, two passes over a register-resident row (one warp per row)
__global__ void row_stats_kernel(const bf16* __restrict__ X, int64_t ldx, int M, int K, float eps, float* __restrict__ stats) {
  const int warp = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (warp >= M) return;
  const bf16* row = X + (size_t)warp * ldx;
  float s = 0.f;
  for (int k = lane; k < K; k += 32) s += __bfloat162float(row[k]);
  const float mean = warp_sum(s) / (float)K;
  float q = 0.f;
  for (int k = lane; k < K; k += 32) { const float d = __bfloat162float(row[k]) - mean; q = fmaf(d, d, q); }
  const float var = warp_sum(q) / (float)K;
  if (lane == 0) { stats[2 * warp] = mean; stats[2 * warp + 1] = rsqrtf(var + eps); }
}

// mma-fragment order (gemm.cu pack_matrix_bf16_kernel) -> row-major [N][K]
__global__ void unpack_fragments_kernel(const bf16* __restrict__ frag, bf16* __restrict__ dst, int64_t N, int K) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * K) return;
  const int64_t n = i / K, k = i - n * K;
  const int64_t nt = n >> 3, g = n & 7, kt = k >> 5, kk = k & 31;
  const int j = (int)(kk >> 4), c = (int)(kk & 15), half = c >> 3, t = (c & 7) >> 1, e = c & 1;
  const int lane = (int)g * 4 + t, reg = j * 2 + half;
  dst[i] = frag[((nt * (K >> 5) + kt) * 32 + lane) * 8 + reg * 2 + e];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
  }
  return fn;
}
// 2-D bf16 matrix [rows][cols] (cols contiguous, row pitch = cols), box {64, box_rows}, 128-byte swizzle, zero OOB fill
static int make_map(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint32_t box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return fail(PTTS_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)K_STAGE, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(PTTS_ECUDA, "cuTensorMapEncodeTiled failed (%d) dims %llu x %llu box rows %u", (int)r, (unsigned long long)rows, (unsigned long long)cols, box_rows);
  return PTTS_OK;
}

static int pick_ntile(int N) {
  if (N % 128 == 0) return 128;
  if (N % 96 == 0) return 96;
  if (N % 64 == 0) return 64;
  return 32;
}

template <int NT>
static int launch_tile(const CUtensorMap& mx, const CUtensorMap& mw, const Args& p, cudaStream_t st) {
  const size_t smem = wg::smem_bytes<NT>(2 * NT * (int)sizeof(float));
  static bool attr = false;
  if (!attr) {
    PTTS_CHECK_CUDA(cudaFuncSetAttribute(linear_tc_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  dim3 grid((p.M + M_TILE - 1) / M_TILE, p.N / NT, 1);
  linear_tc_kernel<NT><<<grid, wg::THREADS, smem, st>>>(mx, mw, p);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

}  // namespace gtc

bool linear_tc_supported(const LinearArgs& a) {
  return a.M >= gtc::M_TILE && a.K % gtc::K_STAGE == 0 && a.N % 32 == 0 && a.ldx == a.K && a.ldy == a.N && (a.R == nullptr || a.ldr == a.N) &&
         a.epi != EPI_F32;
}

// a: as for launch_linear (bf16); w_rowmajor: the SAME matrix as a.W but row-major [N][K]; stats_scratch: float[2*M] (used when a.c1 != nullptr)
int launch_linear_tc(const LinearArgs& a, const void* w_rowmajor, float* stats_scratch, cudaStream_t st) {
  using namespace gtc;
  Args p{};
  p.M = a.M; p.N = a.N; p.K = a.K;
  const int n_tile = pick_ntile(a.N);
  p.epi = a.epi; p.act = a.act; p.R = (const bf16*)a.R; p.Y = (bf16*)a.Y;
  if (a.c1 != nullptr) {
    const int warps_per_block = 8;
    row_stats_kernel<<<(a.M + warps_per_block - 1) / warps_per_block, warps_per_block * 32, 0, st>>>((const bf16*)a.X, a.ldx, a.M, a.K, a.eps, stats_scratch);
    PTTS_LAUNCH_CHECK();
    p.stats = stats_scratch; p.c1 = a.c1; p.c2 = a.c2;
  }
  CUtensorMap mx, mw;
  if (int e = make_map(&mx, a.X, (uint64_t)a.K, (uint64_t)a.M, (uint32_t)M_TILE)) return e;
  if (int e = make_map(&mw, w_rowmajor, (uint64_t)a.K, (uint64_t)a.N, (uint32_t)n_tile)) return e;
  switch (n_tile) {
    case 128: return launch_tile<128>(mx, mw, p, st);
    case 96: return launch_tile<96>(mx, mw, p, st);
    case 64: return launch_tile<64>(mx, mw, p, st);
    default: return launch_tile<32>(mx, mw, p, st);
  }
}

int unpack_fragments(const void* frag, void* dst_rowmajor, int64_t N, int K, cudaStream_t st) {
  const int64_t n = N * K;
  gtc::unpack_fragments_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>((const bf16*)frag, (bf16*)dst_rowmajor, N, K);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

}  // namespace ptts
