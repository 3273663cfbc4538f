// dac.cu -- DAC codec decode: codebook ids -> latent -> waveform.
//
// Replaces DACModel.decode (parler_tts/dac_wrapper/modeling_dac.py:106-142), i.e. the two calls into
// descript-audio-codec: quantizer.from_codes (:138) and model.decode (:139).  Arithmetic restated from
// transformers' DacModel (models/dac/modeling_dac.py:345-369 from_codes, :405-440 decoder, :234-262
// block, :173-207 residual unit, :85-99 snake); weight-norm is folded at load (reference :148-157).
//
// Layout: activations are channels-last [B][T][C] so one time step's channels are contiguous (the
// implicit-GEMM K dimension) -- the reference's cuDNN path is channels-first.
// This file is the generic fp32-accumulate implicit-GEMM path (any channel count, any dtype):
// one kernel covers Conv1d(k=7, dilated), Conv1d(k=1) and ConvTranspose1d(k=2s, stride s) by
// describing each as "n_taps shifted input rows x per-tap weight slice"; snake on the input, bias,
// residual add and tanh are fused.  Roofline: tensor/FMA-bound (1.608 GFLOP per code frame, SURVEY 8d).
// dac_decode at the end walks the codec's layers by name (dac.h) on this path or on the wgmma one (dac_tc.cu).
#include <utility>
#include <vector>

#include "common.cuh"
#include "dac.h"

namespace ptts {

// snake(x) = x + (alpha + 1e-9)^-1 * sin(alpha x)^2, every op rounded to the storage dtype like torch.
template <typename T>
__device__ __forceinline__ float snake_fn(float x, float alpha, float inv) {
  const float s = DT<T>::rnd(sinf(DT<T>::rnd(alpha * x)));
  return DT<T>::rnd(x + DT<T>::rnd(inv * DT<T>::rnd(s * s)));
}

constexpr int CT_M = 64, CT_N = 64, CT_K = 16, CT_AROWS = 128, CT_MAXTAPS = 7;

// SAMPLES: a ragged encode's lengths (RowLengths, hop > 0).  WINDOW: a windowed decode (RowLengths::emit_lo), whose rows outside
// needed_rows are written as 0 and whose tiles without a needed row skip the K loop.
template <typename T, bool SAMPLES, bool WINDOW = false>
__global__ void __launch_bounds__(256) conv_kernel(ConvArgs p, RowLengths rl) {
  __shared__ float As[CT_K][CT_AROWS];
  __shared__ __align__(16) float Bs[CT_MAXTAPS][CT_K][CT_N];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int phase = blockIdx.z % p.n_phase, b = blockIdx.z / p.n_phase;
  const int q0 = blockIdx.x * CT_M, co0 = blockIdx.y * CT_N;
  const int wt_base = p.wt_base + phase * p.wt_phase_step;
  // input row window of this tile: q0 + off_lo .. q0 + CT_M - 1 + off_hi
  const int off_last = p.off_base + (p.n_taps - 1) * p.off_step;
  const int off_lo = min(p.off_base, off_last);
  // this row's lengths: a ragged decode loads its input as if the buffer ended at the row's end (the zero padding a standalone
  // decode sees) and writes 0 past its output end; a tile wholly past the end skips the K loop
  int t_in = p.Tin, t_out = p.Tout, q_end = p.q_count;
  if (rl.frame_lengths != nullptr) {
    const int n = row_frames<SAMPLES>(rl.frame_lengths, b, rl.frames, rl.hop);
    t_in = n * rl.up_in; t_out = n * rl.up_out; q_end = p.q_count - p.Tin + t_in;
  }
  int2 need = make_int2(0, 0);
  if constexpr (WINDOW) {
    need = needed_rows(rl.emit_lo, rl.emit_hi, b, row_frames(rl.frame_lengths, b, rl.frames), rl.up_out, rl.m_lo, rl.m_hi);
    const int to0 = q0 * p.o_mul + p.o_add + phase * p.o_phase_step;
    if (to0 + (CT_M - 1) * p.o_mul < need.x || to0 >= need.y) q_end = q0;
  }
  const T* __restrict__ x = reinterpret_cast<const T*>(p.x) + (size_t)b * p.Tin * p.Cin;
  const T* __restrict__ w = reinterpret_cast<const T*>(p.w);
  const T* __restrict__ alpha = reinterpret_cast<const T*>(p.alpha);
  const int arows = CT_M + abs(off_last - p.off_base);

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

  for (int ci0 = 0; q0 < q_end && ci0 < p.Cin; ci0 += CT_K) {
    __syncthreads();
    // A tile: (snake of) x[q0+off_lo+r][ci0+c], zero outside [0,Tin) -- conv zero padding
    for (int e = tid; e < arows * CT_K; e += 256) {
      const int r = e / CT_K, c = e - r * CT_K;
      const int t = q0 + off_lo + r, ci = ci0 + c;
      float v = 0.f;
      if (t >= 0 && t < t_in && ci < p.Cin) {
        v = DT<T>::to_f(x[(size_t)t * p.Cin + ci]);
        if (alpha != nullptr) {
          const float a = DT<T>::to_f(alpha[ci]);
          v = snake_fn<T>(v, a, DT<T>::rnd(1.0f / DT<T>::rnd(a + 1e-9f)));
        }
      }
      As[c][r] = v;
    }
    // B tile: w[tap][ci0+c][co0+n]
    for (int e = tid; e < p.n_taps * CT_K * CT_N; e += 256) {
      const int n = e % CT_N, c = (e / CT_N) % CT_K, j = e / (CT_N * CT_K);
      const int ci = ci0 + c, co = co0 + n;
      float v = 0.f;
      if (ci < p.Cin && co < p.Cout) v = DT<T>::to_f(w[((size_t)(wt_base + j * p.wt_step) * p.Cin + ci) * p.Cout + co]);
      Bs[j][c][n] = v;
    }
    __syncthreads();
    for (int j = 0; j < p.n_taps; j++) {
      const int roff = p.off_base + j * p.off_step - off_lo;
#pragma unroll
      for (int c = 0; c < CT_K; c++) {
        const float4 bv = *reinterpret_cast<const float4*>(&Bs[j][c][tx * 4]);
        float av[4];
#pragma unroll
        for (int i = 0; i < 4; i++) av[i] = As[c][ty * 4 + i + roff];
#pragma unroll
        for (int i = 0; i < 4; i++) {
          acc[i][0] = fmaf(av[i], bv.x, acc[i][0]);
          acc[i][1] = fmaf(av[i], bv.y, acc[i][1]);
          acc[i][2] = fmaf(av[i], bv.z, acc[i][2]);
          acc[i][3] = fmaf(av[i], bv.w, acc[i][3]);
        }
      }
    }
  }
  const T* __restrict__ bias = reinterpret_cast<const T*>(p.bias);
  const T* __restrict__ res = reinterpret_cast<const T*>(p.res);
  T* __restrict__ out = reinterpret_cast<T*>(p.out);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int q = q0 + ty * 4 + i;
    if (q >= p.q_count) continue;
    const int to = q * p.o_mul + p.o_add + phase * p.o_phase_step;
    if (to < 0 || to >= p.Tout) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int co = co0 + tx * 4 + j;
      if (co >= p.Cout) continue;
      const size_t o = ((size_t)b * p.Tout + to) * p.Cout + co;
      if (to >= t_out || (WINDOW && (to < need.x || to >= need.y))) { out[o] = DT<T>::from_f(0.f); continue; }
      float v = DT<T>::rnd(acc[i][j] + DT<T>::to_f(bias[co]));
      if (res != nullptr) v = DT<T>::rnd(DT<T>::to_f(res[o]) + v);
      if (p.tanh_out) v = tanhf(v);
      out[o] = DT<T>::from_f(v);
    }
  }
}

int launch_conv(const ConvArgs& a, int dtype, int B, cudaStream_t st, const RowLengths& rl) {
  PTTS_REQUIRE(a.n_taps >= 1 && a.n_taps <= CT_MAXTAPS, "conv: n_taps %d out of range", a.n_taps);
  PTTS_REQUIRE(CT_M + abs((a.n_taps - 1) * a.off_step) <= CT_AROWS, "conv: receptive field too wide");
  dim3 grid((a.q_count + CT_M - 1) / CT_M, (a.Cout + CT_N - 1) / CT_N, B * a.n_phase);
  const bool samples = rl.frame_lengths != nullptr && rl.hop > 0;
  if (rl.emit_lo != nullptr) {
    PTTS_REQUIRE(rl.frame_lengths != nullptr && !samples, "conv: a windowed decode needs frame lengths");
    (dtype == PTTS_BF16 ? conv_kernel<bf16, false, true> : conv_kernel<float, false, true>)<<<grid, 256, 0, st>>>(a, rl);
  } else if (dtype == PTTS_BF16) (samples ? conv_kernel<bf16, true> : conv_kernel<bf16, false>)<<<grid, 256, 0, st>>>(a, rl);
  else (samples ? conv_kernel<float, true> : conv_kernel<float, false>)<<<grid, 256, 0, st>>>(a, rl);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// quantizer.from_codes: z[b][t][c] = sum_k ( out_proj_k.bias[c] + sum_d out_proj_k.w[c][d] * codebook_k[code][d] )
// accumulated codebook by codebook in the storage dtype (quantized_representation += ..., :367).
template <typename T, bool WINDOW = false>   // WINDOW: a windowed decode (FromCodesArgs::emit_lo)
__global__ void __launch_bounds__(256) from_codes_kernel(FromCodesArgs p) {
  __shared__ float e[32][16];  // [k][d] for this (b, t)
  const int t = blockIdx.x, b = blockIdx.y;
  const int K = p.K, D = p.D;
  int src = t;   // code frame of latent frame t
  if constexpr (WINDOW) {
    const int n = row_frames(p.frame_lengths, b, p.T);
    const int2 need = needed_rows(p.emit_lo, p.emit_hi, b, n, 1, p.m_lo, p.m_hi);
    if (t < need.x || t >= need.y) return;                                  // not needed: left as it is
    src = min(max(__ldg(p.frame_start + b), 0), p.codes_T - n) + t;         // n <= T <= codes_T (host-checked)
  }
  if (p.frame_lengths != nullptr && t >= row_frames(p.frame_lengths, b, p.T)) {   // past a ragged row's end: a zero latent
    T* __restrict__ z = reinterpret_cast<T*>(p.z) + ((size_t)b * p.T + t) * p.C;
    for (int c = threadIdx.x; c < p.C; c += blockDim.x) z[c] = DT<T>::from_f(0.f);
    return;
  }
  if (threadIdx.x < K * D) {
    const int k = threadIdx.x / D, d = threadIdx.x - k * D;
    const int64_t code = p.codes[((size_t)b * K + k) * (WINDOW ? p.codes_T : p.T) + src];
    e[k][d] = DT<T>::to_f(reinterpret_cast<const T*>(p.codebooks)[((size_t)k * p.codebook_size + code) * D + d]);
  }
  __syncthreads();
  const T* __restrict__ W = reinterpret_cast<const T*>(p.proj_w);
  const T* __restrict__ Bv = reinterpret_cast<const T*>(p.proj_b);
  T* __restrict__ z = reinterpret_cast<T*>(p.z) + ((size_t)b * p.T + t) * p.C;
  for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < K; k++) {
      float s = 0.f;
      for (int d = 0; d < D; d++) s = fmaf(DT<T>::to_f(W[((size_t)k * p.C + c) * D + d]), e[k][d], s);
      s = DT<T>::rnd(s + DT<T>::to_f(Bv[(size_t)k * p.C + c]));
      acc = (k == 0) ? s : DT<T>::rnd(acc + s);
    }
    z[c] = DT<T>::from_f(acc);
  }
}
int launch_from_codes(const FromCodesArgs& a, int dtype, int B, cudaStream_t st) {
  PTTS_REQUIRE(a.K <= 32 && a.D <= 16 && a.K * a.D <= 256, "from_codes: K=%d D=%d unsupported", a.K, a.D);
  dim3 grid(a.T, B);
  if (a.emit_lo != nullptr) {
    PTTS_REQUIRE(a.frame_lengths != nullptr && a.frame_start != nullptr && a.T <= a.codes_T, "from_codes: bad window arguments");
    (dtype == PTTS_BF16 ? from_codes_kernel<bf16, true> : from_codes_kernel<float, true>)<<<grid, 256, 0, st>>>(a);
  } else if (dtype == PTTS_BF16) from_codes_kernel<bf16><<<grid, 256, 0, st>>>(a);
  else from_codes_kernel<float><<<grid, 256, 0, st>>>(a);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// ---- weight repack: Conv1d [co][ci][k] / ConvTranspose1d [ci][co][k] -> [k][ci][co] ---------------
template <typename S, typename D>
__global__ void pack_conv_kernel(const S* src, D* dst, int d0, int d1, int k, int transposed) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n = (int64_t)d0 * d1 * k;
  if (i >= n) return;
  const int kk = (int)(i % k);
  const int b1 = (int)((i / k) % d1), b0 = (int)(i / ((int64_t)k * d1));
  // conv: (b0,b1)=(co,ci); convT: (b0,b1)=(ci,co)
  const int ci = transposed ? b0 : b1, co = transposed ? b1 : b0;
  const int Cin = transposed ? d0 : d1, Cout = transposed ? d1 : d0;
  float v;
  if constexpr (sizeof(S) == 2) v = __bfloat162float(src[i]); else v = src[i];
  const size_t o = ((size_t)kk * Cin + ci) * Cout + co;
  if constexpr (sizeof(D) == 2) dst[o] = __float2bfloat16_rn(v); else dst[o] = v;
}
int pack_conv(const void* src, int src_dtype, void* dst, int dst_dtype, int d0, int d1, int k, int transposed, cudaStream_t st) {
  const int64_t n = (int64_t)d0 * d1 * k;
  const int blocks = (int)((n + 255) / 256);
  if (src_dtype == PTTS_BF16 && dst_dtype == PTTS_BF16) pack_conv_kernel<bf16, bf16><<<blocks, 256, 0, st>>>((const bf16*)src, (bf16*)dst, d0, d1, k, transposed);
  else if (src_dtype == PTTS_BF16) pack_conv_kernel<bf16, float><<<blocks, 256, 0, st>>>((const bf16*)src, (float*)dst, d0, d1, k, transposed);
  else if (dst_dtype == PTTS_BF16) pack_conv_kernel<float, bf16><<<blocks, 256, 0, st>>>((const float*)src, (bf16*)dst, d0, d1, k, transposed);
  else pack_conv_kernel<float, float><<<blocks, 256, 0, st>>>((const float*)src, (float*)dst, d0, d1, k, transposed);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// audio [B][T][1] is already [B, 1, T] contiguous: nothing to transpose for the final layer.


// ---- output convolution: Conv1d(C -> 1, k = 7) + tanh on the channels-last, already snake'd tensor ----------------------------
// The generic tile kernel above computes a 64 x 64 output tile: with ONE output channel 63/64 of its FMAs are wasted.
// Here one thread owns one output sample: the 128 + 6 input rows of a block are staged in shared memory (row pitch padded to
// C + 8 elements so that 8 consecutive threads' 16-byte reads hit 8 different bank groups), weights [7][C] as fp32.
// bf16 inputs, fp32 accumulation in tap-major / channel order, one rounding of acc + bias, tanh, one rounding (torch's ops).
constexpr int FC_T = 128;   // outputs per block
template <bool WINDOW = false>   // WINDOW: a windowed decode, samples outside the emit range [emit_lo, emit_hi) are 0
__global__ void __launch_bounds__(FC_T) final_conv_tanh_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, const bf16* __restrict__ bias,
                                                               bf16* __restrict__ out, int C, int T,
                                                               const int32_t* __restrict__ frame_lengths, int frames,
                                                               const int32_t* __restrict__ emit_lo, const int32_t* __restrict__ emit_hi) {
  extern __shared__ __align__(16) unsigned char fsm[];
  const int pitch = C + 8;                                   // elements
  bf16* xs = reinterpret_cast<bf16*>(fsm);                   // [FC_T + 6][pitch]
  float* ws = reinterpret_cast<float*>(fsm + (size_t)(FC_T + 6) * pitch * 2);   // [7][C]
  const int b = blockIdx.y, t0 = blockIdx.x * FC_T, tid = threadIdx.x;
  // a ragged row's samples end at n_b * hop: later samples are 0 (not tanh(bias)); a block wholly past the end loads nothing.
  // Inputs up to 3 rows past the end are read by kept samples: the zero band the last conv wrote there.
  int t_end = frame_lengths != nullptr ? row_frames(frame_lengths, b, frames) * (T / frames) : T;
  int t_beg = 0;
  if constexpr (WINDOW) {   // the emit range: the only samples computed, and they read only rows the convs before computed
    const int2 need = needed_rows(emit_lo, emit_hi, b, row_frames(frame_lengths, b, frames), T / frames, 0, 0);
    t_beg = need.x; t_end = need.y;
  }
  if (t0 >= t_end || (WINDOW && t0 + FC_T <= t_beg)) {
    if (t0 + tid < T) out[(size_t)b * T + t0 + tid] = __float2bfloat16_rn(0.f);
    return;
  }
  const bf16* xb = x + (size_t)b * T * C;
  const int vec_per_row = C / 8;
  for (int e = tid; e < (FC_T + 6) * vec_per_row; e += FC_T) {
    const int r = e / vec_per_row, c = e - r * vec_per_row;
    const int t = t0 - 3 + r;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);                    // zero padding outside [0, T)
    if (t >= 0 && t < T) v = *reinterpret_cast<const uint4*>(xb + (size_t)t * C + c * 8);
    *reinterpret_cast<uint4*>(xs + (size_t)r * pitch + c * 8) = v;
  }
  for (int e = tid; e < 7 * C; e += FC_T) ws[e] = __bfloat162float(w[e]);   // packed [tap][Cin][Cout = 1]
  __syncthreads();
  const int t = t0 + tid;
  if (t >= T) return;
  float acc = 0.f;
  for (int j = 0; j < 7; j++) {
    const bf16* row = xs + (size_t)(tid + j) * pitch;
    const float* wj = ws + j * C;
    for (int c = 0; c < C; c += 8) {
      float v[8];
      load8(row + c, v);
#pragma unroll
      for (int e = 0; e < 8; e++) acc = fmaf(v[e], wj[c + e], acc);
    }
  }
  const float y = DT<bf16>::rnd(acc + __bfloat162float(bias[0]));
  out[(size_t)b * T + t] = __float2bfloat16_rn(t < t_end && (!WINDOW || t >= t_beg) ? tanhf(y) : 0.f);
}

bool final_conv_supported(int C) { return C % 8 == 0 && C <= 512; }
int launch_final_conv_tanh(const void* x, const void* w, const void* bias, void* out, int C, int T, int B, const int32_t* frame_lengths,
                           int frames, cudaStream_t st, const int32_t* emit_lo, const int32_t* emit_hi) {
  const size_t smem = (size_t)(FC_T + 6) * (C + 8) * 2 + (size_t)7 * C * 4;
  static bool attr = false;
  if (!attr) {
    PTTS_CHECK_CUDA(cudaFuncSetAttribute(final_conv_tanh_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    PTTS_CHECK_CUDA(cudaFuncSetAttribute(final_conv_tanh_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attr = true;
  }
  const bool window = emit_lo != nullptr;
  PTTS_REQUIRE(!window || (frame_lengths != nullptr && emit_hi != nullptr), "final conv: a windowed decode needs frame lengths");
  (window ? final_conv_tanh_kernel<true> : final_conv_tanh_kernel<false>)<<<dim3((T + FC_T - 1) / FC_T, B), FC_T, smem, st>>>(
      (const bf16*)x, (const bf16*)w, (const bf16*)bias, (bf16*)out, C, T, frame_lengths, frames, emit_lo, emit_hi);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// ---- decode walk: from_codes into the latent buffer, then conv1, the decoder blocks and the output conv ----------------------
// Each conv gets its row lengths as time steps per code frame so far (Tin / T, Tout / T), which place each ragged row's end.
static const int kDilation[3] = {1, 3, 9};

// Windowed decode: the rows each layer must compute beyond [lo * up, hi * up) on its output axis, so that the samples of the emit
// frames [lo, hi) come out as in a whole decode.  Walked backwards from the output conv (margins 0): a stride-1 conv with taps k,
// dilation d reads (k - 1) / 2 * d rows on each side; the transposed conv's output row q * s - pad + p reads input rows q and
// q - 1 (conv_up), so output rows [A, C) read input rows [floor((A + pad) / s) - 1, floor((C - 1 + pad) / s)].  The residual
// path adds nothing (its reach is 0).  Same interval arithmetic as incremental.dac_dependency_radius; exact up to the transposed
// conv's rounding, which only widens.  Returns [from_codes (latent frames), conv 1, ..., output conv], in walk order.
struct Margin { int lo, hi; };
static int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }
static std::vector<Margin> window_margins(const ptts_dac_config& c) {
  std::vector<Margin> m;
  Margin cur{0, 0};
  auto same = [&](int taps, int dil) { m.push_back(cur); cur = {cur.lo + (taps - 1) / 2 * dil, cur.hi + (taps - 1) / 2 * dil}; };
  same(7, 1);                                              // output conv
  for (int bi = c.n_blocks - 1; bi >= 0; bi--) {
    const int s = c.strides[bi], pad = (s + 1) / 2;
    for (int r = 2; r >= 0; r--) { same(1, 1); same(7, kDilation[r]); }
    m.push_back(cur);                                      // transposed conv
    cur = {1 - floor_div(pad - cur.lo, s), floor_div(cur.hi - 1 + pad, s) + 1};
  }
  same(7, 1);                                              // conv 1
  m.push_back(cur);                                        // from_codes
  return std::vector<Margin>(m.rbegin(), m.rend());
}

// Each conv's RowLengths in walk order; in a windowed decode (win != nullptr) with its margins.
struct WalkRows {
  const int32_t* fl;
  int T;
  const DacWindow* win;
  std::vector<Margin> m;
  size_t i = 1;   // m[0] is from_codes'
  RowLengths next(int up_in, int up_out) {
    RowLengths r{fl, T, up_in, up_out};
    if (win != nullptr) { r.emit_lo = win->emit_lo; r.emit_hi = win->emit_hi; r.m_lo = m[i].lo; r.m_hi = m[i].hi; }
    i++;
    return r;
  }
};

// bf16, every conv but the last (Cout = 1) as a wgmma implicit GEMM.  Snake moves into the epilogue of the conv before it: a conv
// writes its raw output where a residual needs it and snake_{alpha of the next layer}(output) for the next conv to read.
static int decode_tc(const ptts_dac_config& c, const DacLayout& L, const char* bl, const DacWorkspace& W, void* ws, int B, int T,
                     WalkRows& rows, void* audio, cudaStream_t st) {
  auto P = [&](int i) { return (const void*)(bl + L.t[i].off); };
  auto conv = [&](ConvArgs a, const void* x, int w, int b, const void* res, void* out_raw, void* out_act, const void* alpha_next) {
    a.x = x; a.bias = P(b); a.res = res;
    return launch_conv_tc(a, bl + L.t[w].off_k, a.n_taps * a.n_phase, alpha_next, out_raw, out_act, B, st, rows.next(a.Tin / T, a.Tout / T));
  };
  char* act = W.buf(ws, 0);   // snake'd input of the next conv
  char* oth = W.buf(ws, 1);
  char* res = W.buf(ws, 2);   // residual stream of the current block
  const int C = c.decoder_dim, nb = c.n_blocks;
  if (int e = conv(conv_same(c.latent_dim, C, T, 7, 1), W.buf(ws, 3), L.conv1_w, L.conv1_b, nullptr, nullptr, act, P(L.block[0].snake1))) return e;
  int Tl = T;
  for (int bi = 0; bi < nb; bi++) {
    const DacDecBlock& blk = L.block[bi];
    const int cout = C >> (bi + 1), s = c.strides[bi];
    if (int e = conv(conv_up(C >> bi, cout, Tl, s), act, blk.conv_t1_w, blk.conv_t1_b, nullptr, res, oth, P(blk.res[0].snake1))) return e;
    std::swap(act, oth);
    Tl *= s;
    for (int r = 0; r < 3; r++) {
      const DacResUnit& u = blk.res[r];
      const int next = r < 2 ? blk.res[r + 1].snake1 : bi + 1 < nb ? L.block[bi + 1].snake1 : L.snake1;
      // y = conv7(snake1(x)): only snake2(y) is stored; x += conv1(snake2(y)), and snake_next(x) for the next layer
      if (int e = conv(conv_same(cout, cout, Tl, 7, kDilation[r]), act, u.conv1_w, u.conv1_b, nullptr, nullptr, oth, P(u.snake2))) return e;
      if (int e = conv(conv_same(cout, cout, Tl, 1, 1), oth, u.conv2_w, u.conv2_b, res, res, act, P(next))) return e;
    }
  }
  const int cl = C >> nb;
  const RowLengths rl = rows.next(Tl / T, Tl / T);
  if (final_conv_supported(cl))   // one thread per output sample
    return launch_final_conv_tanh(act, P(L.conv2_w), P(L.conv2_b), audio, cl, Tl, B, rl.frame_lengths, T, st, rl.emit_lo, rl.emit_hi);
  ConvArgs f = conv_same(cl, 1, Tl, 7, 1);   // the input is already snake'd
  f.x = act; f.w = P(L.conv2_w); f.bias = P(L.conv2_b); f.out = audio; f.tanh_out = 1;
  return launch_conv(f, c.dtype, B, st, rl);
}

// Any dtype and width: snake applied on the fly to each conv's input, the residual added in place.
static int decode_generic(const ptts_dac_config& c, const DacLayout& L, const char* bl, const DacWorkspace& W, void* ws, int B, int T,
                          WalkRows& rows, void* audio, cudaStream_t st) {
  auto P = [&](int i) { return (const void*)(bl + L.t[i].off); };
  auto conv = [&](ConvArgs a, const void* x, const void* alpha, int w, int b, const void* res, void* out) {
    a.x = x; a.alpha = alpha; a.w = P(w); a.bias = P(b); a.res = res; a.out = out;
    return launch_conv(a, c.dtype, B, st, rows.next(a.Tin / T, a.Tout / T));
  };
  char* cur = W.buf(ws, 0);
  char* oth = W.buf(ws, 1);
  const int C = c.decoder_dim;
  if (int e = conv(conv_same(c.latent_dim, C, T, 7, 1), W.buf(ws, 3), nullptr, L.conv1_w, L.conv1_b, nullptr, cur)) return e;
  int Tl = T;
  for (int bi = 0; bi < c.n_blocks; bi++) {
    const DacDecBlock& blk = L.block[bi];
    const int cout = C >> (bi + 1), s = c.strides[bi];
    if (int e = conv(conv_up(C >> bi, cout, Tl, s), cur, P(blk.snake1), blk.conv_t1_w, blk.conv_t1_b, nullptr, oth)) return e;
    std::swap(cur, oth);
    Tl *= s;
    for (int r = 0; r < 3; r++) {
      const DacResUnit& u = blk.res[r];
      // y = conv7(snake1(x)) -> oth; x = x + conv1(snake2(y)) in place
      if (int e = conv(conv_same(cout, cout, Tl, 7, kDilation[r]), cur, P(u.snake1), u.conv1_w, u.conv1_b, nullptr, oth)) return e;
      if (int e = conv(conv_same(cout, cout, Tl, 1, 1), oth, P(u.snake2), u.conv2_w, u.conv2_b, cur, cur)) return e;
    }
  }
  ConvArgs f = conv_same(C >> c.n_blocks, 1, Tl, 7, 1);
  f.tanh_out = 1;
  return conv(f, cur, P(L.snake1), L.conv2_w, L.conv2_b, nullptr, audio);
}

static int decode_walk(const ptts_dac_config& c, const void* blob, void* ws, const int64_t* codes, int B, int T, const int32_t* frame_lengths,
                       const DacWindow* win, void* audio, bool allow_tc, cudaStream_t st) {
  const DacLayout L = make_dac_layout(c);
  const DacWorkspace W = dac_decode_workspace(c, B, T);
  const char* bl = (const char*)blob;
  WalkRows rows{frame_lengths, T, win, win != nullptr ? window_margins(c) : std::vector<Margin>{}};
  FromCodesArgs fz{codes, bl + L.codebooks, bl + L.proj_w, bl + L.proj_b, W.buf(ws, 3), c.n_codebooks, c.codebook_dim, c.latent_dim, T,
                   c.codebook_size, frame_lengths};
  if (win != nullptr) {
    fz.frame_start = win->frame_start; fz.emit_lo = win->emit_lo; fz.emit_hi = win->emit_hi;
    fz.codes_T = win->codes_T; fz.m_lo = rows.m[0].lo; fz.m_hi = rows.m[0].hi;
  }
  if (int e = launch_from_codes(fz, c.dtype, B, st)) return e;
  bool tc = allow_tc && c.dtype == PTTS_BF16 && conv_tc_supported(c.latent_dim, c.decoder_dim);
  for (int bi = 0; bi < c.n_blocks && tc; bi++) {
    const int cin = c.decoder_dim >> bi, cout = c.decoder_dim >> (bi + 1);
    tc = conv_tc_supported(cin, cout) && conv_tc_supported(cout, cout);
  }
  return (tc ? decode_tc : decode_generic)(c, L, bl, W, ws, B, T, rows, audio, st);
}

int dac_decode(const ptts_dac_config& c, const void* blob, void* ws, const int64_t* codes, int B, int T, const int32_t* frame_lengths,
               void* audio, bool allow_tc, cudaStream_t st) {
  return decode_walk(c, blob, ws, codes, B, T, frame_lengths, nullptr, audio, allow_tc, st);
}

int dac_decode_window(const ptts_dac_config& c, const void* blob, void* ws, const int64_t* codes, int B, int T, const int32_t* frame_lengths,
                      const DacWindow& win, void* audio, bool allow_tc, cudaStream_t st) {
  return decode_walk(c, blob, ws, codes, B, T, frame_lengths, &win, audio, allow_tc, st);
}

}  // namespace ptts
