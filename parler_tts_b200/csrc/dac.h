// dac.h -- DAC decode and encode: kernel argument structs, blob layouts and tensor tables.
#pragma once
#include <vector>
#include "common.cuh"
#include "layout.h"

namespace ptts {

// One launch of the generic implicit-GEMM kernel.  Output row of tile row q (per phase):
//   to = q*o_mul + o_add + phase*o_phase_step;   input row for tap j: q + off_base + j*off_step;
//   weight slice for tap j: wt_base + phase*wt_phase_step + j*wt_step   (weights are [tap][Cin][Cout]).
struct ConvArgs {
  const void* x; const void* w; const void* bias; const void* alpha; const void* res; void* out;
  int Cin, Cout, Tin, Tout, q_count;
  int n_taps, off_base, off_step, wt_base, wt_step;
  int n_phase, wt_phase_step, o_mul, o_add, o_phase_step;
  int tanh_out;
};
// The codec's three conv shapes: geometry only, the caller sets the pointers.  Their weights hold n_taps * n_phase taps.
// Stride-1 Conv1d(k = taps, dilation dil, "same" padding) over T rows.
static inline ConvArgs conv_same(int Cin, int Cout, int T, int taps, int dil) {
  ConvArgs a{};
  a.Cin = Cin; a.Cout = Cout; a.Tin = T; a.Tout = T; a.q_count = T;
  a.n_taps = taps; a.off_base = -((taps - 1) / 2) * dil; a.off_step = dil; a.wt_base = 0; a.wt_step = 1;
  a.n_phase = 1; a.wt_phase_step = 0; a.o_mul = 1; a.o_add = 0; a.o_phase_step = 0;
  return a;
}
// ConvTranspose1d(k = 2s, stride s, pad ceil(s/2)) from T rows to T*s: phase p of output row q*s - pad + p takes taps p and
// p + s at input rows q and q - 1.
static inline ConvArgs conv_up(int Cin, int Cout, int T, int s) {
  ConvArgs a{};
  a.Cin = Cin; a.Cout = Cout; a.Tin = T; a.Tout = T * s; a.q_count = T + 1;
  a.n_taps = 2; a.off_base = 0; a.off_step = -1; a.wt_base = 0; a.wt_step = s;
  a.n_phase = s; a.wt_phase_step = 1; a.o_mul = s; a.o_add = -((s + 1) / 2); a.o_phase_step = 1;
  return a;
}
// The encoder's strided Conv1d(C -> Cout, k = 2s, stride s) over T rows: the 3-tap conv over super-rows q-1, q, q+1 of the
// [B][T/s][s*C] view (pack_strided_conv below).
static inline ConvArgs conv_super_rows(int C, int Cout, int T, int s) { return conv_same(s * C, Cout, T / s, 3, 1); }

// Ragged batch: row b holds n_b code frames and ends at n_b * up_in on a conv's input axis, * up_out on its output axis.  Outputs
// past a row's end are written as 0, so that the buffers hold the zero padding a standalone run of the row sees.
//   hop == 0 (decode): n_b = frame_lengths[b], clamped to [0, frames];
//   hop > 0 (encode):  frame_lengths[b] counts waveform samples, clamped to [1, frames * hop]; n_b = ceil(samples / hop).
// frame_lengths == nullptr: every row is full (equal lengths).
// Windowed decode (emit_lo != nullptr, hop == 0): the conv computes only the output rows [lo_b * up_out - m_lo, hi_b * up_out + m_hi)
// of row b, the rows the samples of frames [lo_b, hi_b) depend on through the layers after it (needed_rows).
struct RowLengths {
  const int32_t* frame_lengths;
  int frames, up_in, up_out;
  int hop;
  const int32_t* emit_lo; const int32_t* emit_hi;
  int m_lo, m_hi;
};
int launch_conv(const ConvArgs& a, int dtype, int B, cudaStream_t st, const RowLengths& rl = RowLengths{});

// code frames of row b of a ragged decode, clamped to [0, frames] so that no value can move a kernel outside its row
__device__ __forceinline__ int row_frames(const int32_t* frame_lengths, int b, int frames) {
  return min(max(__ldg(frame_lengths + b), 0), frames);
}
// waveform samples of row b of a ragged encode, clamped to [1, samples]
__device__ __forceinline__ int row_samples(const int32_t* sample_lengths, int b, int samples) {
  return min(max(__ldg(sample_lengths + b), 1), samples);
}
// code frames of row b, lengths counting samples (SAMPLES: a ragged encode, hop > 0) or frames.  The kernels that take both are
// instantiated once per reading, so that the decode's instantiations stay the code they were before the encode's.
template <bool SAMPLES>
__device__ __forceinline__ int row_frames(const int32_t* lengths, int b, int frames, int hop) {
  if constexpr (SAMPLES) return (row_samples(lengths, b, frames * hop) + hop - 1) / hop;
  else return row_frames(lengths, b, frames);
}
// The output rows [x, y) of row b (n frames) that a windowed decode needs from a layer with up_out rows per frame: the emit range
// [lo_b, hi_b), clamped to [0, n], widened by the layer's margins.  Rows past n * up_out in it are the zero padding later layers
// read.  An empty emit range needs nothing (x == y).
__device__ __forceinline__ int2 needed_rows(const int32_t* emit_lo, const int32_t* emit_hi, int b, int n, int up_out, int m_lo, int m_hi) {
  const int lo = min(max(__ldg(emit_lo + b), 0), n), hi = min(max(__ldg(emit_hi + b), lo), n);
  if (lo == hi) return make_int2(0, 0);
  return make_int2(lo * up_out - m_lo, hi * up_out + m_hi);
}

struct FromCodesArgs {
  const int64_t* codes;  // [B][K][T]
  const void* codebooks; const void* proj_w; const void* proj_b;  // [K][cs][D], [K][C][D], [K][C]
  void* z;               // [B][T][C]
  int K, D, C, T, codebook_size;
  const int32_t* frame_lengths;  // [B] or nullptr: frames at or past row b's length are zero latents and read no code
  // windowed decode (emit_lo != nullptr): codes are [B][K][codes_T] and latent frame t of row b is code frame frame_start[b] + t;
  // only the frames of needed_rows(m_lo, m_hi) are written
  const int32_t* frame_start; const int32_t* emit_lo; const int32_t* emit_hi;
  int codes_T, m_lo, m_hi;
};
int launch_from_codes(const FromCodesArgs& a, int dtype, int B, cudaStream_t st);
int pack_conv(const void* src, int src_dtype, void* dst, int dst_dtype, int d0, int d1, int k, int transposed, cudaStream_t st);
// tensor-core path (dac_tc.cu, wgmma)
bool conv_tc_supported(int Cin, int Cout);
int launch_conv_tc(const ConvArgs& a, const void* w_kmajor, int taps_total, const void* alpha_next, void* out_raw, void* out_act, int B, cudaStream_t st,
                   const RowLengths& rl = RowLengths{});
int pack_conv_kmajor(const void* src, int src_dtype, void* dst, int d0, int d1, int k, int transposed, cudaStream_t st);
// output convolution (C -> 1, k = 7) + tanh on the already snake'd channels-last tensor, bf16 (dac.cu)
bool final_conv_supported(int C);
// frame_lengths (nullptr: none) as in RowLengths, `frames` code frames of T / frames samples each: samples past a row's end are 0.
// emit_lo / emit_hi (nullptr: none): a windowed decode, samples outside the emit frames [lo_b, hi_b) are 0.
int launch_final_conv_tanh(const void* x, const void* w, const void* bias, void* out, int C, int T, int B, const int32_t* frame_lengths,
                           int frames, cudaStream_t st, const int32_t* emit_lo = nullptr, const int32_t* emit_hi = nullptr);

enum { DK_PLAIN = 0, DK_CONV = 1, DK_CONVT = 2 };
struct DacTensor {
  int kind;
  int d0, d1, k;   // source dims (conv: co,ci,k; convT: ci,co,k; plain: numel,1,1)
  int64_t off;     // byte offset in blob
  int64_t numel;
  int64_t off_k;   // conv weights: second copy [tap][Cout][Cin] bf16 for the tensor-core path (-1: none)
};

// Tensor ids (indices into a layout's t) under the state-dict names of dac_wrapper._dac_tensor_list /
// _dac_encoder_tensor_list; the ids themselves are the push order of make_dac_layout / make_dac_enc_layout.
struct DacResUnit { int snake1, conv1_w, conv1_b, snake2, conv2_w, conv2_b; };
struct DacDecBlock { int snake1, conv_t1_w, conv_t1_b; DacResUnit res[3]; };
struct DacEncBlock { DacResUnit res[3]; int snake1, conv1_w, conv1_b; };

struct DacLayout {
  std::vector<DacTensor> t;
  int64_t codebooks, proj_w, proj_b;
  int conv1_w, conv1_b;
  DacDecBlock block[8];
  int snake1, conv2_w, conv2_b;
  int64_t total;
  int es;
};

static inline int validate_dac(const ptts_dac_config& c) {
  PTTS_REQUIRE(c.dtype == PTTS_BF16 || c.dtype == PTTS_F32, "dac dtype must be bf16 or f32");
  PTTS_REQUIRE(c.n_blocks >= 1 && c.n_blocks <= 8, "dac n_blocks out of range");
  PTTS_REQUIRE(c.n_codebooks >= 1 && c.n_codebooks <= 32 && c.codebook_dim >= 1 && c.codebook_dim <= 16 &&
               c.n_codebooks * c.codebook_dim <= 256, "dac codebook shape unsupported");
  PTTS_REQUIRE((c.decoder_dim >> c.n_blocks) >= 1, "dac decoder_dim too small for n_blocks");
  for (int i = 0; i < c.n_blocks; i++) PTTS_REQUIRE(c.strides[i] >= 1 && c.strides[i] % 2 == 0 && c.strides[i] <= 32, "dac stride %d must be even and <= 32", c.strides[i]);
  return PTTS_OK;
}

static inline DacLayout make_dac_layout(const ptts_dac_config& c) {
  DacLayout L;
  L.es = dtype_size(c.dtype);
  int64_t o = 0;
  auto add = [&](int kind, int d0, int d1, int k) {
    DacTensor t{kind, d0, d1, k, o, (int64_t)d0 * d1 * k, -1};
    o = align_up(o + t.numel * L.es, 256);
    if (kind != DK_PLAIN && c.dtype == PTTS_BF16) { t.off_k = o; o = align_up(o + t.numel * 2, 1024); }
    L.t.push_back(t);
    return (int)L.t.size() - 1;
  };
  const int K = c.n_codebooks, D = c.codebook_dim, Z = c.latent_dim;
  // from_codes tensors are laid out as three contiguous arrays; ids interleave per codebook
  L.codebooks = 0;
  L.proj_w = align_up((int64_t)K * c.codebook_size * D * L.es, 256);
  L.proj_b = L.proj_w + align_up((int64_t)K * Z * D * L.es, 256);
  o = L.proj_b + align_up((int64_t)K * Z * L.es, 256);
  for (int k = 0; k < K; k++) {
    L.t.push_back({DK_PLAIN, c.codebook_size * D, 1, 1, L.codebooks + (int64_t)k * c.codebook_size * D * L.es, (int64_t)c.codebook_size * D, -1});
    L.t.push_back({DK_PLAIN, Z * D, 1, 1, L.proj_w + (int64_t)k * Z * D * L.es, (int64_t)Z * D, -1});
    L.t.push_back({DK_PLAIN, Z, 1, 1, L.proj_b + (int64_t)k * Z * L.es, (int64_t)Z, -1});
  }
  const int C = c.decoder_dim;
  L.conv1_w = add(DK_CONV, C, Z, 7); L.conv1_b = add(DK_PLAIN, C, 1, 1);
  for (int bi = 0; bi < c.n_blocks; bi++) {
    const int cin = C >> bi, cout = C >> (bi + 1), s = c.strides[bi];
    DacDecBlock& b = L.block[bi];
    b.snake1 = add(DK_PLAIN, cin, 1, 1);
    b.conv_t1_w = add(DK_CONVT, cin, cout, 2 * s); b.conv_t1_b = add(DK_PLAIN, cout, 1, 1);
    for (DacResUnit& u : b.res) {
      u.snake1 = add(DK_PLAIN, cout, 1, 1);
      u.conv1_w = add(DK_CONV, cout, cout, 7); u.conv1_b = add(DK_PLAIN, cout, 1, 1);
      u.snake2 = add(DK_PLAIN, cout, 1, 1);
      u.conv2_w = add(DK_CONV, cout, cout, 1); u.conv2_b = add(DK_PLAIN, cout, 1, 1);
    }
  }
  const int cl = C >> c.n_blocks;
  L.snake1 = add(DK_PLAIN, cl, 1, 1);
  L.conv2_w = add(DK_CONV, 1, cl, 7); L.conv2_b = add(DK_PLAIN, 1, 1, 1);
  L.total = o;
  return L;
}

static inline int dac_hop(const ptts_dac_config& c) {
  int h = 1;
  for (int i = 0; i < c.n_blocks; i++) h *= c.strides[i];
  return h;
}

// ---- DAC encode (dac_enc.cu) ----------------------------------------------------------------------
// A strided Conv1d(C -> 2C, k = 2s, stride s, pad s/2) over [B][T][C] is an ordinary 3-tap conv over the [B][T/s][s*C] view
// ("super-rows" q-1, q, q+1; tap j, in-row offset r carries weight tap r + j*s - s/2 when that lies in [0, 2s), else 0).
// kmajor != 0: [3][Cout][s*C] bf16 (wgmma path); else [3][s*C][Cout] in dst_dtype (generic conv_kernel).
int pack_strided_conv(const void* src, int src_dtype, void* dst, int dst_dtype, int Cout, int C, int s, int kmajor, cudaStream_t st);
// codebook [n][D] (rounded to bf16 first when round_bf16) -> rows / max(||row||, 1e-12) in fp32 (F.normalize)
int pack_normalized_codebook(const void* src, int src_dtype, float* dst, int n, int D, int round_bf16, cudaStream_t st);
// Conv1d(1 -> C, k = 7, pad 3) over the waveform [B][samples] (zero beyond `samples`, T rows out, bf16): raw [B][T][C] and
// snake_{alpha_next}(raw) for the next layer -- the wgmma kernel needs Cin >= 64.  sample_lengths (nullptr: none), a ragged
// encode as in RowLengths with T / hop frames: row b reads no sample past its own count and ends at ceil(count / hop) * hop rows;
// it writes zeros over more than conv_tc_kernel's 128-row zero band past that end.
int launch_enc_input_conv(const void* audio, const void* w, const void* bias, const void* alpha_next, void* out_raw, void* out_act,
                          int C, int samples, int T, int B, const int32_t* sample_lengths, int hop, cudaStream_t st);
struct QuantizeArgs {
  void* z;                // [B][T][Z] encoder output (frames past a ragged row's end are set to 0)
  const void* in_w;       // [K][D][Z]
  const void* in_b;       // [K][D]
  const float* cb_norm;   // [K][cs][D] fp32, unit rows
  const void* codebooks;  // [K][cs][D] raw (decode blob)
  const void* out_w;      // [K][Z][D] (decode blob)
  const void* out_b;      // [K][Z]   (decode blob)
  int64_t* codes;         // [B][n_q][T]
  int n_q, D, Z, T, codebook_size;
  const int32_t* sample_lengths;   // [B] or nullptr: a ragged encode (RowLengths, hop > 0); frames past a row's end code as
  int hop;                         // codebook_size and read no latent
};
bool quantize_supported(int Z, int D);
int launch_quantize(const QuantizeArgs& a, int dtype, int B, cudaStream_t st);

// Encoder tensor table (ptts_dac_encoder_pack ids): dac_wrapper.py::_dac_encoder_tensor_list gives the state-dict keys.
enum { EK_PLAIN = 0, EK_CONV = 1, EK_SCONV = 2, EK_CODEBOOK = 3 };
struct DacEncTensor {
  int kind;
  int d0, d1, k;   // conv: co, ci, k; plain / codebook: numel or rows, 1 / D, 1
  int tile;        // plain: > 1 also stores the vector tiled `tile` times at off_t (snake before a strided conv, generic path)
  int64_t off, numel;
  int64_t off_k;   // conv weights, bf16 config: [tap][Cout][Cin] k-major copy (strided: the super-row form) for wgmma; -1: none
  int64_t off_t;
};
struct DacEncLayout {
  std::vector<DacEncTensor> t;
  int64_t in_w, in_b, cb_norm;   // quantizer arrays, contiguous over codebooks
  int conv1_w, conv1_b;
  DacEncBlock block[8];
  int snake1, conv2_w, conv2_b;
  int64_t total;
  int es;
};

static inline int validate_dac_encoder(const ptts_dac_config& c) {
  if (int e = validate_dac(c)) return e;
  PTTS_REQUIRE(c.encoder_dim > 0, "dac config has no encoder (encoder_dim = 0: decode only)");
  PTTS_REQUIRE(c.n_enc_blocks >= 1 && c.n_enc_blocks <= 8, "dac encoder block count %d out of range", c.n_enc_blocks);
  int hop = 1;
  for (int i = 0; i < c.n_enc_blocks; i++) {
    PTTS_REQUIRE(c.encoder_rates[i] >= 2 && c.encoder_rates[i] % 2 == 0 && c.encoder_rates[i] <= 32,
                 "dac encoder stride %d must be even and <= 32", c.encoder_rates[i]);
    hop *= c.encoder_rates[i];
  }
  PTTS_REQUIRE(hop == dac_hop(c), "dac encoder hop %d differs from the decoder hop %d", hop, dac_hop(c));
  PTTS_REQUIRE(((int64_t)c.encoder_dim << c.n_enc_blocks) <= 65536, "dac encoder_dim too large");
  // refused here rather than at the quantizer's launch, after the whole encoder network has run
  PTTS_REQUIRE(quantize_supported(c.latent_dim, c.codebook_dim),
               "dac quantizer: latent_dim %d / codebook_dim %d unsupported (codebook_dim 4, 8 or 16, latent_dim 1..1536)", c.latent_dim,
               c.codebook_dim);
  return PTTS_OK;
}

static inline DacEncLayout make_dac_enc_layout(const ptts_dac_config& c) {
  DacEncLayout L;
  L.es = dtype_size(c.dtype);
  const int K = c.n_codebooks, D = c.codebook_dim, Z = c.latent_dim, cs = c.codebook_size;
  L.in_w = 0;
  L.in_b = align_up((int64_t)K * D * Z * L.es, 256);
  L.cb_norm = L.in_b + align_up((int64_t)K * D * L.es, 256);
  int64_t o = L.cb_norm + align_up((int64_t)K * cs * D * 4, 256);
  const bool tc = c.dtype == PTTS_BF16;
  auto add = [&](int kind, int d0, int d1, int k, int tile) {
    DacEncTensor t{kind, d0, d1, k, tile, o, (int64_t)d0 * d1 * k, -1, -1};
    // a strided conv's generic copy is the [3][s*C][Cout] super-row form: 1.5x the source weight
    const int64_t stored = kind == EK_SCONV ? (int64_t)3 * d0 * d1 * (k / 2) : t.numel;
    o = align_up(o + stored * L.es, 256);
    if (tc && (kind == EK_SCONV || (kind == EK_CONV && d1 > 1))) { t.off_k = o; o = align_up(o + stored * 2, 1024); }
    if (tile > 1) { t.off_t = o; o = align_up(o + t.numel * tile * L.es, 256); }
    L.t.push_back(t);
    return (int)L.t.size() - 1;
  };
  L.conv1_w = add(EK_CONV, c.encoder_dim, 1, 7, 1); L.conv1_b = add(EK_PLAIN, c.encoder_dim, 1, 1, 1);
  for (int bi = 0; bi < c.n_enc_blocks; bi++) {
    const int C = c.encoder_dim << bi, s = c.encoder_rates[bi];
    DacEncBlock& b = L.block[bi];
    for (DacResUnit& u : b.res) {
      u.snake1 = add(EK_PLAIN, C, 1, 1, 1);
      u.conv1_w = add(EK_CONV, C, C, 7, 1); u.conv1_b = add(EK_PLAIN, C, 1, 1, 1);
      u.snake2 = add(EK_PLAIN, C, 1, 1, 1);
      u.conv2_w = add(EK_CONV, C, C, 1, 1); u.conv2_b = add(EK_PLAIN, C, 1, 1, 1);
    }
    b.snake1 = add(EK_PLAIN, C, 1, 1, s);
    b.conv1_w = add(EK_SCONV, 2 * C, C, 2 * s, 1); b.conv1_b = add(EK_PLAIN, 2 * C, 1, 1, 1);
  }
  const int cf = c.encoder_dim << c.n_enc_blocks;
  L.snake1 = add(EK_PLAIN, cf, 1, 1, 1);
  L.conv2_w = add(EK_CONV, Z, cf, 3, 1); L.conv2_b = add(EK_PLAIN, Z, 1, 1, 1);
  for (int k = 0; k < K; k++) {
    L.t.push_back({EK_PLAIN, D * Z, 1, 1, 1, L.in_w + (int64_t)k * D * Z * L.es, (int64_t)D * Z, -1, -1});
    L.t.push_back({EK_PLAIN, D, 1, 1, 1, L.in_b + (int64_t)k * D * L.es, (int64_t)D, -1, -1});
    L.t.push_back({EK_CODEBOOK, cs, D, 1, 1, L.cb_norm + (int64_t)k * cs * D * 4, (int64_t)cs * D, -1, -1});
  }
  L.total = o;
  return L;
}

// Codec workspace: three activation buffers, each of the largest activation (per_frame elements per batch row and code frame),
// then the latent [B][T][latent_dim].  T: code frames (encode: samples rounded up to the hop).
struct DacWorkspace {
  int64_t act, z;   // bytes of one activation buffer, of the latent buffer
  int64_t bytes() const { return 3 * act + z; }
  char* buf(void* ws, int i) const { return (char*)ws + i * act; }   // activation buffer i; i = 3: the latent
};
static inline DacWorkspace dac_workspace(const ptts_dac_config& c, int64_t per_frame, int B, int64_t T) {
  const int64_t es = dtype_size(c.dtype);
  return {align_up(per_frame * B * T * es, 1024), align_up((int64_t)c.latent_dim * B * T * es, 1024)};
}
static inline DacWorkspace dac_decode_workspace(const ptts_dac_config& c, int B, int T) {
  int64_t m = c.latent_dim > c.decoder_dim ? c.latent_dim : c.decoder_dim, up = 1;
  for (int i = 0; i < c.n_blocks; i++) {
    up *= c.strides[i];
    const int64_t e = up * (c.decoder_dim >> (i + 1));
    if (e > m) m = e;
  }
  return dac_workspace(c, m, B, T);
}
static inline DacWorkspace dac_encode_workspace(const ptts_dac_config& c, int B, int samples) {
  int64_t per = dac_hop(c), m = (int64_t)c.latent_dim;
  for (int bi = 0; bi <= c.n_enc_blocks; bi++) {
    const int64_t e = per * ((int64_t)c.encoder_dim << bi);
    if (e > m) m = e;
    if (bi < c.n_enc_blocks) per /= c.encoder_rates[bi];
  }
  return dac_workspace(c, m, B, (samples + dac_hop(c) - 1) / dac_hop(c));
}

// codes [B][K][T] -> waveform [B][T * hop] (dac.cu).  frame_lengths as in RowLengths.  allow_tc: the wgmma path where the config
// is bf16 and conv_tc_supported takes every width; the generic conv_kernel path otherwise.
int dac_decode(const ptts_dac_config& c, const void* blob, void* ws, const int64_t* codes, int B, int T, const int32_t* frame_lengths,
               void* audio, bool allow_tc, cudaStream_t st);
// Windowed decode (ptts_dac_decode3): row b decodes code frames [frame_start[b], + frame_lengths[b]) of codes [B][K][codes_T] as
// dac_decode decodes them alone at frame 0, and keeps the samples of frames [emit_lo[b], emit_hi[b]) (the rest are 0).  Each
// layer computes only the rows those samples depend on (window_margins in dac.cu).
struct DacWindow {
  const int32_t* frame_start; const int32_t* emit_lo; const int32_t* emit_hi;
  int codes_T;
};
int dac_decode_window(const ptts_dac_config& c, const void* blob, void* ws, const int64_t* codes, int B, int T, const int32_t* frame_lengths,
                      const DacWindow& win, void* audio, bool allow_tc, cudaStream_t st);
// waveform [B][samples] -> codes [B][n_q][T] and, when latents != nullptr, the encoder output [B][T][latent_dim] (dac_enc.cu).
// sample_lengths (device [B], or nullptr: every row has `samples`): a ragged encode whose row b equals the encode of its first
// sample_lengths[b] samples alone in its first ceil(sample_lengths[b] / hop) frames; later frames hold codebook_size and zero
// latents.  allow_tc as for dac_decode.
int dac_encode(const ptts_dac_config& c, const void* dec_blob, const void* enc_blob, void* ws, const void* audio, int B, int samples,
               const int32_t* sample_lengths, int n_q, int64_t* codes, void* latents, bool allow_tc, cudaStream_t st);

}  // namespace ptts
