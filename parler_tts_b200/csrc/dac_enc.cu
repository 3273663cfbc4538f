// dac_enc.cu -- DAC codec encode: waveform -> latent -> codebook ids.
//
// Replaces DACModel.encode (parler_tts/dac_wrapper/modeling_dac.py:33-104), i.e. descript-audio-codec's model.preprocess
// (:64, right zero-pad to the hop) and model.encode (:95).  Arithmetic restated from transformers' DacModel
// (models/dac/modeling_dac.py:442-472 encoder, :210-231 block, :173-207 residual unit, :281-343 residual vector quantizer,
// :102-170 vector quantize).  The encoder's residual units and its final k3 conv run on the decode path's conv kernels
// (conv_tc_kernel in dac_tc.cu, conv_kernel in dac.cu); this file adds what those cannot do:
//   * the input conv (Cin = 1; the wgmma kernel needs Cin >= 64),
//   * the weight packs of the strided convs, which run as 3-tap convs over the [B][T/s][s*C] view (dac.h),
//   * the residual vector quantizer,
//   * dac_encode, the walk over the encoder's layers by name (dac.h).
#include <math.h>

#include <utility>

#include "common.cuh"
#include "dac.h"

namespace ptts {

// ---- strided conv weight: [Cout][C][2s] -> the super-row form (dac.h) ----------------------------------------------------
template <typename S, typename D>
__global__ void pack_strided_conv_kernel(const S* __restrict__ src, D* __restrict__ dst, int Cout, int C, int s, int kmajor) {
  const int64_t sc = (int64_t)s * C;
  const int64_t n = 3 * sc * Cout;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t cip; int co, j;
  if (kmajor) { cip = i % sc; co = (int)((i / sc) % Cout); j = (int)(i / (sc * Cout)); }
  else { co = (int)(i % Cout); cip = (i / Cout) % sc; j = (int)(i / (sc * Cout)); }
  const int r = (int)(cip / C), ci = (int)(cip - (int64_t)r * C);
  const int k = r + j * s - s / 2;
  float v = 0.f;
  if (k >= 0 && k < 2 * s) {
    const S w = src[((int64_t)co * C + ci) * (2 * s) + k];
    if constexpr (sizeof(S) == 2) v = __bfloat162float(w); else v = w;
  }
  if constexpr (sizeof(D) == 2) dst[i] = __float2bfloat16_rn(v); else dst[i] = v;
}
int pack_strided_conv(const void* src, int src_dtype, void* dst, int dst_dtype, int Cout, int C, int s, int kmajor, cudaStream_t st) {
  const int64_t n = (int64_t)3 * s * C * Cout;
  const int blocks = (int)((n + 255) / 256);
  if (src_dtype == PTTS_BF16 && dst_dtype == PTTS_BF16) pack_strided_conv_kernel<bf16, bf16><<<blocks, 256, 0, st>>>((const bf16*)src, (bf16*)dst, Cout, C, s, kmajor);
  else if (src_dtype == PTTS_BF16) pack_strided_conv_kernel<bf16, float><<<blocks, 256, 0, st>>>((const bf16*)src, (float*)dst, Cout, C, s, kmajor);
  else if (dst_dtype == PTTS_BF16) pack_strided_conv_kernel<float, bf16><<<blocks, 256, 0, st>>>((const float*)src, (bf16*)dst, Cout, C, s, kmajor);
  else pack_strided_conv_kernel<float, float><<<blocks, 256, 0, st>>>((const float*)src, (float*)dst, Cout, C, s, kmajor);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// ---- codebook rows -> unit rows in fp32 (F.normalize in decode_latents, :160-161) ----------------------------------------
template <typename S>
__global__ void pack_normalized_codebook_kernel(const S* __restrict__ src, float* __restrict__ dst, int n, int D, int round_bf16) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n) return;
  auto f = [&](int d) {   // the codebook as the model holds it (bf16 model: rounded to bf16), then normalised in fp32
    const S v = src[(int64_t)row * D + d];
    float x;
    if constexpr (sizeof(S) == 2) x = __bfloat162float(v); else x = (float)v;
    return round_bf16 ? __bfloat162float(__float2bfloat16_rn(x)) : x;
  };
  float ss = 0.f;
  for (int d = 0; d < D; d++) ss = fmaf(f(d), f(d), ss);
  const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
  for (int d = 0; d < D; d++) dst[(int64_t)row * D + d] = f(d) * inv;
}
int pack_normalized_codebook(const void* src, int src_dtype, float* dst, int n, int D, int round_bf16, cudaStream_t st) {
  const int blocks = (n + 255) / 256;
  if (src_dtype == PTTS_BF16) pack_normalized_codebook_kernel<bf16><<<blocks, 256, 0, st>>>((const bf16*)src, dst, n, D, round_bf16);
  else pack_normalized_codebook_kernel<float><<<blocks, 256, 0, st>>>((const float*)src, dst, n, D, round_bf16);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// ---- input conv: Conv1d(1 -> C, k = 7, pad 3) on the bf16 waveform --------------------------------------------------------
// One block covers IC_ROWS output rows x all C channels; its waveform window and the [7][C] weights sit in shared memory.  Each
// thread writes channel pairs, with the same bf16x2 epilogue as conv_tc_kernel: raw = bf16(acc + bias) (taps summed in order
// 0..6 in fp32), act = raw + inv * sin(alpha * raw)^2 for the next layer.
// A ragged row (sample_lengths) reads n_b samples and computes rows [0, t_end), t_end = ceil(n_b / hop) * hop, the rows of its
// standalone encode.  Rows [t_end, t_end + ZERO_BAND] are written as 0: the zero padding the next conv_tc_kernel reads (its
// reach past a row's end is at most its 128-row tile, host-checked there); blocks past that band exit.
constexpr int IC_ROWS = 64, ZERO_BAND = 128;
__global__ void __launch_bounds__(256) enc_input_conv_kernel(const bf16* __restrict__ audio, const bf16* __restrict__ w, const bf16* __restrict__ bias,
                                                             const bf16* __restrict__ alpha_next, bf16* __restrict__ out_raw, bf16* __restrict__ out_act,
                                                             int C, int samples, int T, const int32_t* __restrict__ sample_lengths, int hop) {
  extern __shared__ float icm[];
  float* xs = icm;                    // [IC_ROWS + 6] waveform window
  float* ws = xs + IC_ROWS + 8;       // [7][C]
  __nv_bfloat162* chan = reinterpret_cast<__nv_bfloat162*>(ws + 7 * C);   // [3][C/2]: bias | alpha | 1/(alpha + 1e-9)
  const int b = blockIdx.y, t0 = blockIdx.x * IC_ROWS, tid = threadIdx.x, half = C / 2;
  int n = samples, t_end = T;
  if (sample_lengths != nullptr) {
    n = row_samples(sample_lengths, b, samples);
    t_end = (n + hop - 1) / hop * hop;
    if (t0 > t_end + ZERO_BAND) return;
  }
  for (int e = tid; e < IC_ROWS + 6; e += blockDim.x) {
    const int t = t0 - 3 + e;
    xs[e] = (t >= 0 && t < n) ? __bfloat162float(audio[(size_t)b * samples + t]) : 0.f;   // conv padding + the pad to the hop
  }
  for (int e = tid; e < 7 * C; e += blockDim.x) ws[e] = __bfloat162float(w[e]);
  for (int c = tid; c < half; c += blockDim.x) {
    const __nv_bfloat162 a = reinterpret_cast<const __nv_bfloat162*>(alpha_next)[c];
    const float2 af = __bfloat1622float2(a);
    chan[c] = reinterpret_cast<const __nv_bfloat162*>(bias)[c];
    chan[half + c] = a;
    chan[2 * half + c] = __floats2bfloat162_rn(1.0f / __bfloat162float(__float2bfloat16_rn(af.x + 1e-9f)),
                                               1.0f / __bfloat162float(__float2bfloat16_rn(af.y + 1e-9f)));
  }
  __syncthreads();
  for (int e = tid; e < IC_ROWS * half; e += blockDim.x) {
    const int r = e / half, cp = e - r * half, t = t0 + r;
    if (t >= T) break;
    const size_t o = ((size_t)b * T + t) * C + 2 * cp;
    if (t >= t_end) {   // past a ragged row's end: raw 0 and snake(0) = 0
      *reinterpret_cast<__nv_bfloat162*>(out_raw + o) = __floats2bfloat162_rn(0.f, 0.f);
      *reinterpret_cast<__nv_bfloat162*>(out_act + o) = __floats2bfloat162_rn(0.f, 0.f);
      continue;
    }
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int j = 0; j < 7; j++) {
      const float x = xs[r + j];
      a0 = fmaf(x, ws[j * C + 2 * cp], a0);
      a1 = fmaf(x, ws[j * C + 2 * cp + 1], a1);
    }
    const float2 bb = __bfloat1622float2(chan[cp]);
    const __nv_bfloat162 r2 = __floats2bfloat162_rn(a0 + bb.x, a1 + bb.y);
    *reinterpret_cast<__nv_bfloat162*>(out_raw + o) = r2;
    const __nv_bfloat162 ax = __hmul2(chan[half + cp], r2);
    const float2 axf = __bfloat1622float2(ax);
    const __nv_bfloat162 sn = __floats2bfloat162_rn(__sinf(axf.x), __sinf(axf.y));
    // __hmul2_rn keeps the product's own rounding (torch's): a plain __hmul2 followed by __hadd2 is contracted into an fma
    *reinterpret_cast<__nv_bfloat162*>(out_act + o) = __hadd2(r2, __hmul2_rn(chan[2 * half + cp], __hmul2(sn, sn)));
  }
}
int launch_enc_input_conv(const void* audio, const void* w, const void* bias, const void* alpha_next, void* out_raw, void* out_act,
                          int C, int samples, int T, int B, const int32_t* sample_lengths, int hop, cudaStream_t st) {
  PTTS_REQUIRE(C % 2 == 0 && C <= 4096, "dac encode: input conv width %d unsupported", C);
  PTTS_REQUIRE(sample_lengths == nullptr || (hop > 0 && T % hop == 0 && samples <= T), "dac encode: ragged input conv needs T = frames * hop");
  const size_t smem = (size_t)(IC_ROWS + 8 + 7 * C) * 4 + (size_t)3 * C * 2;
  static bool attr = false;
  if (!attr) { PTTS_CHECK_CUDA(cudaFuncSetAttribute(enc_input_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024)); attr = true; }
  enc_input_conv_kernel<<<dim3((T + IC_ROWS - 1) / IC_ROWS, B), 256, smem, st>>>((const bf16*)audio, (const bf16*)w, (const bf16*)bias,
                                                                                (const bf16*)alpha_next, (bf16*)out_raw, (bf16*)out_act, C, samples, T,
                                                                                sample_lengths, hop);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// ---- residual vector quantizer (DacResidualVectorQuantizer.forward, :320-338) --------------------------------------------
// One warp per code frame, all n_q codebooks in turn; lane l owns latent channels l, l + 32, ... of the residual (shared
// memory), so in_proj and the residual update need no exchange beyond the D warp sums of in_proj.  Per codebook:
//   z_e = in_proj(residual)                                  bf16(acc + bias) like torch's 1x1 conv
//   code = argmax_c <z_e / |z_e|, c_hat>                     fp32, c_hat normalised at pack time; ties -> lowest index
//   (with unit rows, -(|e|^2 - 2 e.c) + |c|^2 = 2 e.c: the reference's distance ranks the codes by this cosine)
//   st = z_e + (z_q - z_e)                                   the straight-through expression, each op rounded (:149)
//   residual -= out_proj(st)                                 bf16(acc + bias), then the rounded difference (:331)
constexpr int QZ_WARPS = 8;
// RAGGED (a ragged encode, p.sample_lengths): frames past a row's end do no work, they write the invalid-frame code codebook_size
// in every codebook (what compact_valid_frames and the decode's range check take as no frame) and a zero latent.
template <typename T, int D, bool RAGGED>
__global__ void __launch_bounds__(QZ_WARPS * 32) quantize_kernel(QuantizeArgs p, int n_frames) {
  extern __shared__ float qres[];   // [QZ_WARPS][Z]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * QZ_WARPS + warp;
  if (f >= n_frames) return;
  const int Z = p.Z, cs = p.codebook_size;
  if constexpr (RAGGED) {
    const int b = f / p.T, t = f - b * p.T;
    if (t >= row_frames<true>(p.sample_lengths, b, p.T, p.hop)) {
      for (int k = lane; k < p.n_q; k += 32) p.codes[((size_t)b * p.n_q + k) * p.T + t] = cs;
      for (int c = lane; c < Z; c += 32) reinterpret_cast<T*>(p.z)[(size_t)f * Z + c] = DT<T>::from_f(0.f);
      return;
    }
  }
  float* r = qres + (size_t)warp * Z;
  const T* z = reinterpret_cast<const T*>(p.z) + (size_t)f * Z;
  for (int c = lane; c < Z; c += 32) r[c] = DT<T>::to_f(z[c]);
  const int b = f / p.T, t = f - b * p.T;
  for (int k = 0; k < p.n_q; k++) {
    const T* W = reinterpret_cast<const T*>(p.in_w) + (size_t)k * D * Z;
    float e[D];
#pragma unroll
    for (int d = 0; d < D; d++) e[d] = 0.f;
    for (int c = lane; c < Z; c += 32) {
      const float rc = r[c];
#pragma unroll
      for (int d = 0; d < D; d++) e[d] = fmaf(DT<T>::to_f(W[(size_t)d * Z + c]), rc, e[d]);
    }
    float n2 = 0.f;
#pragma unroll
    for (int d = 0; d < D; d++) {
      e[d] = DT<T>::rnd(warp_sum(e[d]) + DT<T>::to_f(reinterpret_cast<const T*>(p.in_b)[k * D + d]));
      n2 = fmaf(e[d], e[d], n2);
    }
    const float inv = 1.0f / fmaxf(sqrtf(n2), 1e-12f);
    float en[D];
#pragma unroll
    for (int d = 0; d < D; d++) en[d] = e[d] * inv;
    const float* cb = p.cb_norm + (size_t)k * cs * D;
    float best = -INFINITY;
    int bi = cs;
    for (int j = lane; j < cs; j += 32) {
      const float4* row = reinterpret_cast<const float4*>(cb + (size_t)j * D);
      float s = 0.f;
#pragma unroll
      for (int q = 0; q < D / 4; q++) {
        const float4 v = row[q];
        s = fmaf(en[4 * q], v.x, s); s = fmaf(en[4 * q + 1], v.y, s);
        s = fmaf(en[4 * q + 2], v.z, s); s = fmaf(en[4 * q + 3], v.w, s);
      }
      if (s > best) { best = s; bi = j; }   // j rises: the first of equal values stays
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (bi >= cs) bi = 0;   // every similarity NaN (a NaN latent): the reference's max() would not pick a valid row either
    if (lane == 0) p.codes[((size_t)b * p.n_q + k) * p.T + t] = bi;
    const T* zq = reinterpret_cast<const T*>(p.codebooks) + ((size_t)k * cs + bi) * D;
    float st[D];
#pragma unroll
    for (int d = 0; d < D; d++) st[d] = DT<T>::rnd(e[d] + DT<T>::rnd(DT<T>::to_f(zq[d]) - e[d]));
    const T* Wo = reinterpret_cast<const T*>(p.out_w) + (size_t)k * Z * D;
    const T* bo = reinterpret_cast<const T*>(p.out_b) + (size_t)k * Z;
    for (int c = lane; c < Z; c += 32) {
      float q = 0.f;
#pragma unroll
      for (int d = 0; d < D; d++) q = fmaf(DT<T>::to_f(Wo[(size_t)c * D + d]), st[d], q);
      q = DT<T>::rnd(q + DT<T>::to_f(bo[c]));
      r[c] = DT<T>::rnd(r[c] - q);
    }
  }
}

bool quantize_supported(int Z, int D) { return (D == 4 || D == 8 || D == 16) && Z >= 1 && Z <= 1536; }
template <typename T, bool RAGGED>
static int launch_quantize_t(const QuantizeArgs& a, int B, cudaStream_t st) {
  const int n = B * a.T;
  const size_t smem = (size_t)QZ_WARPS * a.Z * 4;
  dim3 grid((n + QZ_WARPS - 1) / QZ_WARPS);
  if (a.D == 4) quantize_kernel<T, 4, RAGGED><<<grid, QZ_WARPS * 32, smem, st>>>(a, n);
  else if (a.D == 8) quantize_kernel<T, 8, RAGGED><<<grid, QZ_WARPS * 32, smem, st>>>(a, n);
  else quantize_kernel<T, 16, RAGGED><<<grid, QZ_WARPS * 32, smem, st>>>(a, n);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}
int launch_quantize(const QuantizeArgs& a, int dtype, int B, cudaStream_t st) {
  PTTS_REQUIRE(quantize_supported(a.Z, a.D), "dac encode: quantizer shape latent %d / codebook_dim %d unsupported", a.Z, a.D);
  PTTS_REQUIRE(a.sample_lengths == nullptr || a.hop > 0, "dac encode: ragged quantizer needs the hop");
  if (a.sample_lengths != nullptr) return dtype == PTTS_BF16 ? launch_quantize_t<bf16, true>(a, B, st) : launch_quantize_t<float, true>(a, B, st);
  return dtype == PTTS_BF16 ? launch_quantize_t<bf16, false>(a, B, st) : launch_quantize_t<float, false>(a, B, st);
}

// ---- encode walk: the input conv, the encoder blocks, the output conv, the quantizer ---------------------------------------
static const int kDilation[3] = {1, 3, 9};

// Each conv of a ragged encode (sl: sample lengths) gets its rows as time steps per code frame at that layer: hop at full rate,
// then hop / s_0, ... (RowLengths with hop > 0, T frames).
static RowLengths enc_rows(const int32_t* sl, int T, int hop, const ConvArgs& a) {
  return sl != nullptr ? RowLengths{sl, T, a.Tin / T, a.Tout / T, hop} : RowLengths{};
}

// bf16, every conv after the input conv as a wgmma implicit GEMM (the strided ones over the s*C view).  Snake moves into the
// epilogue of the conv before it, as in the decode walk (dac.cu).
static int encode_tc(const ptts_dac_config& c, const DacEncLayout& L, const char* bl, const DacWorkspace& W, void* ws, const void* audio,
                     int B, int samples, const int32_t* sl, int T, void* z, cudaStream_t st) {
  const int hop = dac_hop(c);
  auto P = [&](int i) { return (const void*)(bl + L.t[i].off); };
  auto conv = [&](ConvArgs a, const void* x, int w, int b, const void* res, void* out_raw, void* out_act, const void* alpha_next) {
    a.x = x; a.bias = P(b); a.res = res;
    return launch_conv_tc(a, bl + L.t[w].off_k, a.n_taps * a.n_phase, alpha_next, out_raw, out_act, B, st, enc_rows(sl, T, hop, a));
  };
  char* res = W.buf(ws, 0);   // residual stream of the current block
  char* act = W.buf(ws, 1);   // snake'd input of the next conv
  char* oth = W.buf(ws, 2);
  const int nb = c.n_enc_blocks, C0 = c.encoder_dim;
  int Tl = T * hop;   // samples padded to the hop
  // input conv: raw -> res, snake_{block 0's first snake1}(x) -> act
  if (int e = launch_enc_input_conv(audio, P(L.conv1_w), P(L.conv1_b), P(L.block[0].res[0].snake1), res, act, C0, samples, Tl, B, sl, hop, st))
    return e;
  for (int bi = 0; bi < nb; bi++) {
    const DacEncBlock& blk = L.block[bi];
    const int C = C0 << bi, s = c.encoder_rates[bi];
    for (int r = 0; r < 3; r++) {
      const DacResUnit& u = blk.res[r];
      const int next = r < 2 ? blk.res[r + 1].snake1 : blk.snake1;
      // y = conv7(snake1(x)): only snake2(y) is stored; x += conv1(snake2(y)), and snake_next(x) for the next layer
      if (int e = conv(conv_same(C, C, Tl, 7, kDilation[r]), act, u.conv1_w, u.conv1_b, nullptr, nullptr, oth, P(u.snake2))) return e;
      if (int e = conv(conv_same(C, C, Tl, 1, 1), oth, u.conv2_w, u.conv2_b, res, res, act, P(next))) return e;
    }
    // strided conv; the TMA zero fill of super-rows -1 and T/s is its padding.  Raw -> res (the next block's residual stream; not
    // needed after the last block), snake of the next layer -> oth
    const bool last = bi + 1 == nb;
    const void* alpha_next = P(last ? L.snake1 : L.block[bi + 1].res[0].snake1);
    if (int e = conv(conv_super_rows(C, 2 * C, Tl, s), act, blk.conv1_w, blk.conv1_b, nullptr, last ? nullptr : res, oth, alpha_next)) return e;
    std::swap(act, oth);
    Tl /= s;
  }
  return conv(conv_same(C0 << nb, c.latent_dim, Tl, 3, 1), act, L.conv2_w, L.conv2_b, nullptr, z, nullptr, nullptr);
}

// A ragged batch's waveform with each row's samples past its own count set to 0, [B][T] (the generic walk's input conv reads it)
template <typename S>
__global__ void mask_waveform_kernel(const S* __restrict__ audio, S* __restrict__ out, const int32_t* __restrict__ sample_lengths,
                                     int samples, int T) {
  const int b = blockIdx.y;
  const int n = row_samples(sample_lengths, b, samples);
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < T; t += gridDim.x * blockDim.x)
    out[(size_t)b * T + t] = t < n ? audio[(size_t)b * samples + t] : DT<S>::from_f(0.f);
}

// Any dtype and width: snake applied on the fly to each conv's input, the residual added in place.
static int encode_generic(const ptts_dac_config& c, const DacEncLayout& L, const char* bl, const DacWorkspace& W, void* ws, const void* audio,
                          int B, int samples, const int32_t* sl, int T, void* z, cudaStream_t st) {
  const int hop = dac_hop(c);
  auto P = [&](int i) { return (const void*)(bl + L.t[i].off); };
  auto conv = [&](ConvArgs a, const void* x, const void* alpha, int w, int b, const void* res, void* out) {
    a.x = x; a.alpha = alpha; a.w = P(w); a.bias = P(b); a.res = res; a.out = out;
    return launch_conv(a, c.dtype, B, st, enc_rows(sl, T, hop, a));
  };
  char* cur = W.buf(ws, 0);
  char* oth = W.buf(ws, 2);
  const int nb = c.n_enc_blocks, C0 = c.encoder_dim;
  int Tl = T * hop;   // samples padded to the hop
  ConvArgs in = conv_same(1, C0, Tl, 7, 1);
  if (sl == nullptr) {
    in.Tin = samples;   // rows past `samples` read zeros: the pad to the hop
  } else {
    // a ragged row reads zeros past its own count: the waveform masked into buffer 1 (unused by this walk, and it holds at
    // least C0 * B * Tl elements), read as Tl rows whose end is the row's frames * hop
    char* masked = W.buf(ws, 1);
    const dim3 grid((Tl + 255) / 256 < 64 ? (Tl + 255) / 256 : 64, B);
    if (c.dtype == PTTS_BF16) mask_waveform_kernel<bf16><<<grid, 256, 0, st>>>((const bf16*)audio, (bf16*)masked, sl, samples, Tl);
    else mask_waveform_kernel<float><<<grid, 256, 0, st>>>((const float*)audio, (float*)masked, sl, samples, Tl);
    PTTS_LAUNCH_CHECK();
    audio = masked;
  }
  if (int e = conv(in, audio, nullptr, L.conv1_w, L.conv1_b, nullptr, cur)) return e;
  for (int bi = 0; bi < nb; bi++) {
    const DacEncBlock& blk = L.block[bi];
    const int C = C0 << bi, s = c.encoder_rates[bi];
    for (int r = 0; r < 3; r++) {
      const DacResUnit& u = blk.res[r];
      if (int e = conv(conv_same(C, C, Tl, 7, kDilation[r]), cur, P(u.snake1), u.conv1_w, u.conv1_b, nullptr, oth)) return e;
      if (int e = conv(conv_same(C, C, Tl, 1, 1), oth, P(u.snake2), u.conv2_w, u.conv2_b, cur, cur)) return e;
    }
    // strided conv over the super-row view: the block's snake1 alpha tiled s times matches its s*C input channels
    if (int e = conv(conv_super_rows(C, 2 * C, Tl, s), cur, bl + L.t[blk.snake1].off_t, blk.conv1_w, blk.conv1_b, nullptr, oth)) return e;
    std::swap(cur, oth);
    Tl /= s;
  }
  return conv(conv_same(C0 << nb, c.latent_dim, Tl, 3, 1), cur, P(L.snake1), L.conv2_w, L.conv2_b, nullptr, z);
}

int dac_encode(const ptts_dac_config& c, const void* dec_blob, const void* enc_blob, void* ws, const void* audio, int B, int samples,
               const int32_t* sample_lengths, int n_q, int64_t* codes, void* latents, bool allow_tc, cudaStream_t st) {
  const DacEncLayout L = make_dac_enc_layout(c);
  const DacLayout DL = make_dac_layout(c);
  const DacWorkspace W = dac_encode_workspace(c, B, samples);
  const int nb = c.n_enc_blocks, C0 = c.encoder_dim, Z = c.latent_dim;
  bool tc = allow_tc && c.dtype == PTTS_BF16 && C0 % 2 == 0 && conv_tc_supported(C0 << nb, Z);
  for (int bi = 0; bi < nb && tc; bi++) tc = conv_tc_supported(C0 << bi, C0 << bi) && conv_tc_supported(c.encoder_rates[bi] * (C0 << bi), 2 * (C0 << bi));
  const char* bl = (const char*)enc_blob;
  void* z = latents ? latents : (void*)W.buf(ws, 3);
  const int T = (samples + dac_hop(c) - 1) / dac_hop(c);
  if (int e = (tc ? encode_tc : encode_generic)(c, L, bl, W, ws, audio, B, samples, sample_lengths, T, z, st)) return e;
  const char* dbl = (const char*)dec_blob;
  QuantizeArgs q{z, bl + L.in_w, bl + L.in_b, (const float*)(bl + L.cb_norm), dbl + DL.codebooks, dbl + DL.proj_w, dbl + DL.proj_b,
                 codes, n_q, c.codebook_dim, Z, T, c.codebook_size, sample_lengths, dac_hop(c)};
  return launch_quantize(q, c.dtype, B, st);
}

}  // namespace ptts
