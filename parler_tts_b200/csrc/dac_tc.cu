// dac_tc.cu -- DAC decoder convolutions as Hopper wgmma implicit GEMMs (bf16 operands, fp32 accumulation in registers).
//
// Replaces the cuDNN Conv1d / ConvTranspose1d calls inside dac.model.DAC.decode (reached from
// parler_tts/dac_wrapper/modeling_dac.py:139; arithmetic per transformers/models/dac/modeling_dac.py:173-262).
// Roofline: tensor pipe -- 1.608 GFLOP per code frame (SURVEY 8d); the SIMT path in dac.cu is FMA-bound.
//
// One CTA computes a 128 (time) x N_TILE (output channel) tile:
//   D[t, co] = sum_{tap j} sum_{ci} X[t + off_j, ci] * W[j][co][ci]
//   * activations are channels-last bf16 [B][T][C]: the K dimension (ci) is contiguous, so the A tile of tap j is
//     a plain 3-D TMA box {64 ci, 128 t, 1 b} at row offset off_j; rows outside [0, T) are ZERO-FILLED by the TMA
//     unit, which is exactly the convolution's zero padding (and the channel tail when Cin % 64 != 0);
//   * weights are pre-packed [tap][Cout][Cin] (K-major), B tile = box {64 ci, N_TILE co, 1 tap};
//   * the K loop runs over (tap, 64-channel chunk) pairs through the TMA / wgmma pipeline of wgmma.cuh;
//   * the epilogue adds the bias and the residual to the register accumulators and writes the raw tensor and/or snake(x)
//     for the NEXT layer, so every layer's A operand is a ready-to-MMA bf16 tensor (snake is x + sin^2(alpha x)/(alpha + 1e-9),
//     rounded like torch's bf16 ops).
// ConvTranspose1d(k = 2s, stride s) = s output phases x 2 taps (dac.cu explains the mapping).
#include <algorithm>
#include <type_traits>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "dac.h"
#include "wgmma.cuh"

namespace ptts {

constexpr int TC_M = wg::M_TILE;   // time rows per tile
constexpr int TC_K = wg::K_STAGE;  // ci per pipeline stage

struct ConvTcArgs {
  int Cin, Cout, Tin, Tout, q_count;
  int n_taps, off_base, off_step, wt_base, wt_step;
  int n_phase, wt_phase_step, o_mul, o_add, o_phase_step;
  const bf16* bias;        // [Cout]
  const bf16* res;         // residual (raw tensor, [B][Tout][Cout]) or nullptr
  bf16* out_raw;           // raw result or nullptr
  bf16* out_act;           // snake_{alpha_next}(result) for the next layer or nullptr
  const bf16* alpha_next;  // [Cout]
  const int32_t* frame_lengths;  // ragged batch (RowLengths in dac.h); nullptr: every row is full
  int frames, up_in, up_out, hop;
};
// A windowed decode's launch (RowLengths in dac.h).  A type of its own, so that the other instantiations keep their arguments.
struct ConvTcWindowArgs : ConvTcArgs {
  const int32_t* emit_lo; const int32_t* emit_hi;
  int m_lo, m_hi;
};

// SAMPLES: a ragged encode's lengths (RowLengths, hop > 0).  Args = ConvTcWindowArgs: a windowed decode, whose tiles without a
// row of needed_rows exit before any load.  The rows a kept tile computes outside needed_rows may read stale workspace rows:
// no needed row reads them.
template <int NT, bool SAMPLES, typename Args = ConvTcArgs>
__global__ void __launch_bounds__(wg::THREADS, 2)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, const Args p) {
  constexpr bool WINDOW = std::is_same_v<Args, ConvTcWindowArgs>;
  extern __shared__ unsigned char smem_raw[];
  const wg::Pipe pipe = wg::pipe_setup<NT>(smem_raw);
  bf16* chan = reinterpret_cast<bf16*>(pipe.extra);  // [3][NT]: bias | alpha | 1/(alpha+1e-9)

  const int phase = blockIdx.z % p.n_phase, b = blockIdx.z / p.n_phase;
  const int q0 = blockIdx.x * TC_M, n0 = blockIdx.y * NT;
  const int k_chunks = (p.Cin + TC_K - 1) / TC_K;
  // Ragged batch.  The TMA map zero-fills only past the whole buffer, so a row's zero padding is written instead: every output
  // past the row's end is 0, in the tile that holds the end (q_end) and in the whole tile after it -- a band of more than TC_M
  // positions, wider than any following conv's reach past the end (host-checked).  Tiles past the band exit at once, tiles
  // wholly inside it skip the K loop: the work follows each row's frames, not B * T.
  int n_iter = p.n_taps * k_chunks;
  if (p.frame_lengths != nullptr) {
    const int q_end = p.q_count - p.Tin + row_frames<SAMPLES>(p.frame_lengths, b, p.frames, p.hop) * p.up_in;
    if ((int)blockIdx.x > q_end / TC_M + 1) return;
    if (q0 >= q_end) n_iter = 0;
  }
  if constexpr (WINDOW) {
    const int2 need = needed_rows(p.emit_lo, p.emit_hi, b, row_frames(p.frame_lengths, b, p.frames), p.up_out, p.m_lo, p.m_hi);
    const int to0 = q0 * p.o_mul + p.o_add + phase * p.o_phase_step;
    if (to0 + (TC_M - 1) * p.o_mul < need.x || to0 >= need.y) return;
  }

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
  }
  // per-channel constants of this N tile: bias, alpha, 1/(alpha+1e-9)
  for (int c = threadIdx.x; c < NT; c += blockDim.x) {
    chan[c] = p.bias[n0 + c];
    if (p.out_act != nullptr) {
      const bf16 a = p.alpha_next[n0 + c];
      chan[NT + c] = a;
      chan[2 * NT + c] = __float2bfloat16_rn(1.0f / __bfloat162float(__float2bfloat16_rn(__bfloat162float(a) + 1e-9f)));
    }
  }
  __syncthreads();

  float acc[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; i++) acc[i] = 0.f;
  auto load = [&](int it, unsigned char* a_dst, unsigned char* b_dst, uint64_t* bar) {
    const int j = it / k_chunks, kc = it - j * k_chunks;
    wg::tma_load_3d(a_dst, &map_x, kc * TC_K, q0 + p.off_base + j * p.off_step, b, bar);
    wg::tma_load_3d(b_dst, &map_w, kc * TC_K, n0, p.wt_base + phase * p.wt_phase_step + j * p.wt_step, bar);
  };
  wg::mainloop<NT>(pipe, n_iter, load, acc);
  const int to_end = p.frame_lengths != nullptr ? row_frames<SAMPLES>(p.frame_lengths, b, p.frames, p.hop) * p.up_out : p.Tout;
  if ((threadIdx.x >> 5) == wg::PRODUCER_WARP) {
    // the producer warp, idle now, writes this tile's rows past the row's end: raw 0 (conv(0) + bias is not) and snake(0) = 0
    if (to_end < p.Tout) {
      for (int e = threadIdx.x & 31; e < TC_M * (NT / 8); e += 32) {
        const int q = q0 + e / (NT / 8), c = 8 * (e % (NT / 8));
        const int to = q * p.o_mul + p.o_add + phase * p.o_phase_step;
        if (q >= p.q_count || to < to_end || to >= p.Tout) continue;
        const size_t o = ((size_t)b * p.Tout + to) * p.Cout + n0 + c;
        if (p.out_raw != nullptr) *reinterpret_cast<uint4*>(p.out_raw + o) = make_uint4(0u, 0u, 0u, 0u);
        if (p.out_act != nullptr) *reinterpret_cast<uint4*>(p.out_act + o) = make_uint4(0u, 0u, 0u, 0u);
      }
    }
    return;
  }

  // ===== epilogue: each register pair is two adjacent channels of one time row =====
  const __nv_bfloat162* bias2 = reinterpret_cast<const __nv_bfloat162*>(chan);
  const __nv_bfloat162* alpha2 = reinterpret_cast<const __nv_bfloat162*>(chan + NT);
  const __nv_bfloat162* inv2 = reinterpret_cast<const __nv_bfloat162*>(chan + 2 * NT);
  const int qrow = q0 + 64 * (threadIdx.x >> 7);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int q = qrow + wg::frag_row(2 * h);
    const int to = q * p.o_mul + p.o_add + phase * p.o_phase_step;
    if (q >= p.q_count || to < 0 || to >= to_end) continue;   // to_end <= Tout; the producer warp writes the rows past it
    const size_t orow = ((size_t)b * p.Tout + to) * p.Cout + n0;
#pragma unroll
    for (int j = 0; j < NT / 8; j++) {
      const int i = 4 * j + 2 * h, c = wg::frag_col(i);
      // native bf16x2 arithmetic: every op rounds to bf16 exactly like the torch ops it replaces
      // conv output = bf16(acc + bias) (one rounding of the fp32 sum)
      const float2 bb = __bfloat1622float2(bias2[c >> 1]);
      __nv_bfloat162 r2 = __floats2bfloat162_rn(acc[i] + bb.x, acc[i + 1] + bb.y);
      if (p.res != nullptr) r2 = __hadd2(*reinterpret_cast<const __nv_bfloat162*>(p.res + orow + c), r2);
      if (p.out_raw != nullptr) *reinterpret_cast<__nv_bfloat162*>(p.out_raw + orow + c) = r2;
      if (p.out_act != nullptr) {
        const __nv_bfloat162 ax = __hmul2(alpha2[c >> 1], r2);                        // alpha * x
        const float2 axf = __bfloat1622float2(ax);
        const __nv_bfloat162 sn = __floats2bfloat162_rn(__sinf(axf.x), __sinf(axf.y));  // sin(.)  (MUFU; bf16 result)
        const __nv_bfloat162 sq = __hmul2(sn, sn);                                    // ^2
        *reinterpret_cast<__nv_bfloat162*>(p.out_act + orow + c) = __hadd2(r2, __hmul2_rn(inv2[c >> 1], sq));  // x + inv * sin^2
        // (_rn: the product is rounded before the add, as in torch -- a plain __hmul2 would be contracted into an fma)
      }
    }
  }
}

// ---- host side ----------------------------------------------------------------------------------
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
// 3-D bf16 tensor [d2][d1][d0] (d0 contiguous), box {64, box1, 1}, 128-byte swizzle, zero OOB fill
static int encode_map(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t box1);

// A decode issues ~60 convolution launches over the SAME buffers and shapes every time (the workspace and the weight blob are
// caller-owned and stable): encode each tensor map once and reuse it (cuTensorMapEncodeTiled is a few microseconds of host time
// per call, and a decode makes ~60 of them).
struct MapKey { const void* base; uint64_t d0, d1, d2; uint32_t box1; };
struct MapEntry { MapKey k; CUtensorMap m; };
static int make_map(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t box1) {
  static std::mutex mu;
  static std::vector<MapEntry> cache;
  std::lock_guard<std::mutex> lock(mu);
  for (const MapEntry& e : cache)
    if (e.k.base == base && e.k.d0 == d0 && e.k.d1 == d1 && e.k.d2 == d2 && e.k.box1 == box1) { *m = e.m; return PTTS_OK; }
  if (int e = encode_map(m, base, d0, d1, d2, box1)) return e;
  if (cache.size() >= 4096) cache.clear();   // many distinct (B, T) shapes over a long-lived process: start over
  cache.push_back(MapEntry{MapKey{base, d0, d1, d2, box1}, *m});
  return PTTS_OK;
}
static int encode_map(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t box1) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return fail(PTTS_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {d0 * 2, d0 * d1 * 2};
  cuuint32_t box[3] = {(cuuint32_t)TC_K, box1, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(PTTS_ECUDA, "cuTensorMapEncodeTiled failed (%d) dims %llu %llu %llu box1 %u", (int)r, (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, box1);
  return PTTS_OK;
}

bool conv_tc_supported(int Cin, int Cout) {
  return Cin % 8 == 0 && Cin >= 64 && Cout % 32 == 0 && Cout >= 32;  // row pitch multiple of 16 B; epilogue works in 32-column chunks
}
int conv_tc_ntile(int Cout) {
  if (Cout % 128 == 0) return 128;
  if (Cout % 96 == 0) return 96;
  if (Cout % 64 == 0) return 64;
  return 32;
}

template <int NT, bool SAMPLES, typename Args>
static int launch_conv_tile_t(const CUtensorMap& mx, const CUtensorMap& mw, const Args& p, int B, cudaStream_t st) {
  const size_t smem = wg::smem_bytes<NT>(3 * NT * (int)sizeof(bf16));
  static bool attr = false;
  if (!attr) {
    PTTS_CHECK_CUDA(cudaFuncSetAttribute(conv_tc_kernel<NT, SAMPLES, Args>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  dim3 grid((p.q_count + TC_M - 1) / TC_M, p.Cout / NT, B * p.n_phase);
  conv_tc_kernel<NT, SAMPLES, Args><<<grid, wg::THREADS, smem, st>>>(mx, mw, p);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}
template <int NT>
static int launch_conv_tile(const CUtensorMap& mx, const CUtensorMap& mw, const ConvTcWindowArgs& p, int B, cudaStream_t st) {
  if (p.emit_lo != nullptr) return launch_conv_tile_t<NT, false>(mx, mw, p, B, st);
  const ConvTcArgs& q = p;
  return p.frame_lengths != nullptr && p.hop > 0 ? launch_conv_tile_t<NT, true>(mx, mw, q, B, st) : launch_conv_tile_t<NT, false>(mx, mw, q, B, st);
}

// x: [B][Tin][Cin] bf16, w: [taps_total][Cout][Cin] bf16
int launch_conv_tc(const ConvArgs& a, const void* w_kmajor, int taps_total, const void* alpha_next, void* out_raw, void* out_act, int B, cudaStream_t st,
                   const RowLengths& rl) {
  ConvTcWindowArgs p{};
  p.Cin = a.Cin; p.Cout = a.Cout; p.Tin = a.Tin; p.Tout = a.Tout; p.q_count = a.q_count;
  p.n_taps = a.n_taps; p.off_base = a.off_base; p.off_step = a.off_step; p.wt_base = a.wt_base; p.wt_step = a.wt_step;
  p.n_phase = a.n_phase; p.wt_phase_step = a.wt_phase_step; p.o_mul = a.o_mul; p.o_add = a.o_add; p.o_phase_step = a.o_phase_step;
  const int n_tile = conv_tc_ntile(a.Cout);
  p.bias = (const bf16*)a.bias; p.res = (const bf16*)a.res; p.out_raw = (bf16*)out_raw; p.out_act = (bf16*)out_act; p.alpha_next = (const bf16*)alpha_next;
  p.frame_lengths = rl.frame_lengths; p.frames = rl.frames; p.up_in = rl.up_in; p.up_out = rl.up_out; p.hop = rl.hop;
  p.emit_lo = rl.emit_lo; p.emit_hi = rl.emit_hi; p.m_lo = rl.m_lo; p.m_hi = rl.m_hi;
  if (rl.emit_lo != nullptr) {
    // needed rows past a row's end lie in the zero band the producer warps write (more than TC_M rows): the margin must not pass it
    PTTS_REQUIRE(rl.frame_lengths != nullptr && rl.hop == 0 && rl.emit_hi != nullptr, "conv_tc: a windowed decode needs frame lengths");
    PTTS_REQUIRE(rl.m_hi <= TC_M, "conv_tc: window margin %d rows is wider than the %d-row zero band", rl.m_hi, TC_M);
  }
  if (rl.frame_lengths != nullptr) {
    // a kept output reads this far past its row's end: the highest tap offset, plus the row the transposed conv's extra q reads.
    // The producer of x wrote zeros over more than TC_M positions past the end (for the encoder's super-row convs, more than
    // TC_M rows of the full-rate view, which is more than TC_M / s super-rows: reach 1 needs s <= TC_M, and s <= 32).
    const int reach = std::max(std::max(a.off_base, a.off_base + (a.n_taps - 1) * a.off_step), 0) + (a.q_count - a.Tin);
    PTTS_REQUIRE(reach <= TC_M, "conv_tc: a ragged batch reads %d rows past a row's end, more than the %d-row zero band", reach, TC_M);
    PTTS_REQUIRE(rl.frames > 0 && a.Tin == rl.frames * rl.up_in && a.Tout == rl.frames * rl.up_out, "conv_tc: ragged lengths do not match the shape");
  }
  CUtensorMap mx, mw;
  if (int e = make_map(&mx, a.x, (uint64_t)a.Cin, (uint64_t)a.Tin, (uint64_t)B, TC_M)) return e;
  if (int e = make_map(&mw, w_kmajor, (uint64_t)a.Cin, (uint64_t)a.Cout, (uint64_t)taps_total, (uint32_t)n_tile)) return e;
  switch (n_tile) {
    case 128: return launch_conv_tile<128>(mx, mw, p, B, st);
    case 96: return launch_conv_tile<96>(mx, mw, p, B, st);
    case 64: return launch_conv_tile<64>(mx, mw, p, B, st);
    default: return launch_conv_tile<32>(mx, mw, p, B, st);
  }
}

// weight repack for the tensor-core path: Conv1d [co][ci][k] / ConvTranspose1d [ci][co][k] -> [k][co][ci] bf16
template <typename S>
__global__ void pack_conv_kmajor_kernel(const S* src, bf16* dst, int d0, int d1, int k, int transposed) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n = (int64_t)d0 * d1 * k;
  if (i >= n) return;
  const int kk = (int)(i % k);
  const int b1 = (int)((i / k) % d1), b0 = (int)(i / ((int64_t)k * d1));
  const int ci = transposed ? b0 : b1, co = transposed ? b1 : b0;
  const int Cin = transposed ? d0 : d1, Cout = transposed ? d1 : d0;
  float v;
  if constexpr (sizeof(S) == 2) v = __bfloat162float(src[i]); else v = src[i];
  dst[((size_t)kk * Cout + co) * Cin + ci] = __float2bfloat16_rn(v);
}
int pack_conv_kmajor(const void* src, int src_dtype, void* dst, int d0, int d1, int k, int transposed, cudaStream_t st) {
  const int64_t n = (int64_t)d0 * d1 * k;
  const int blocks = (int)((n + 255) / 256);
  if (src_dtype == PTTS_BF16) pack_conv_kmajor_kernel<bf16><<<blocks, 256, 0, st>>>((const bf16*)src, (bf16*)dst, d0, d1, k, transposed);
  else pack_conv_kmajor_kernel<float><<<blocks, 256, 0, st>>>((const float*)src, (bf16*)dst, d0, d1, k, transposed);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

}  // namespace ptts
