// kernels.h -- host-side launch interface of the kernel translation units.
#pragma once
#include "common.cuh"
#include "layout.h"

namespace ptts {

enum { EPI_STORE = 0, EPI_ACT = 1, EPI_RESIDUAL = 2, EPI_F32 = 3 };

struct LinearArgs {
  const void* X; int64_t ldx;  // activations [M, K], row stride ldx (elements)
  const void* W;               // packed weight slot (fragment order for bf16, row-major for f32)
  void* Y; int64_t ldy;
  const void* R; int64_t ldr;  // residual (EPI_RESIDUAL)
  const float* ln_w; const float* ln_b; float eps;  // fused LayerNorm on x (needs Kc == K); f32 path uses gamma/beta directly
  const float* c1; const float* c2;                 // bf16 path: folded LayerNorm vectors (ln_stats.cuh); LN on iff c1 != nullptr
  int M, N, K, Kc;             // Kc = activation tile width (0 = choose)
  int epi, act;
  const Ctrl* ctrl;            // device control block: kernels no-op once generation has finished
};
int launch_linear(const LinearArgs& a, int dtype, cudaStream_t st, bool pdl, int sm_count);
// wgmma prefill GEMM (gemm_tc.cu): the bf16 prefill's linear layers wherever linear_tc_supported holds
bool linear_tc_supported(const LinearArgs& a);
int launch_linear_tc(const LinearArgs& a, const void* w_rowmajor, float* stats_scratch, cudaStream_t st);
int unpack_fragments(const void* frag, void* dst_rowmajor, int64_t N, int K, cudaStream_t st);
int pack_matrix(const void* src, int src_dtype, int64_t rows, int64_t cols, int row_off, int K, void* dst, int dst_dtype, cudaStream_t st);
int fold_layernorm(void* w_packed, int N, int K, const float* gamma, const float* beta, float* c1, float* c2, cudaStream_t st);
int pack_plain(const void* src, int src_dtype, int64_t n, void* dst, int dst_dtype, cudaStream_t st);

// ---- attention (attention.cu) -------------------------------------------------------------------
struct AttnArgs {
  // query / new-token projections: row r = b*q_len + j of a [B*q_len, ld] matrix
  const void* q; int64_t ldq; int q_col0;       // q head h at columns q_col0 + h*64
  const void* knew; const void* vnew; int64_t ldkv; int k_col0, v_col0;  // self: new K/V rows (same matrix as q)
  void* kcache; void* vcache;                   // self: [B][nkv][Tmax][64]; cross: strided view
  int64_t kv_b_stride, kv_h_stride, kv_t_stride; // element strides of (batch, kv head, token)
  int kv_b_div;         // row b reads the K/V and key-mask rows of batch index b / kv_b_div (cross-attention of a session whose
                        // consecutive rows share one description, ptts_session_create3); 1: its own
  void* out; int64_t ldo;                       // [B*q_len, H]
  const int* key_mask; int mask_len, mask_ld;   // keys t < mask_len with key_mask[b*mask_ld+t]==0 are excluded
  const Ctrl* ctrl;
  int B, nh, nkv, q_len;
  int past_from_ctrl;   // 1: past = prefix + ctrl->cur_len - 1 (decode, less row_shift(shift, b) in attention_decode_kernel); 0: past_len
  int past_len, prefix; // cache position of the first new row
  const int* shift;     // decode: per-row position offsets of a ragged continuation (SampleArgs::shift), or nullptr
  int cross;            // 1: keys = kv_len encoder positions, no append, no causal structure
  int kv_len;
  int rope; const void* rope_cos; const void* rope_sin;  // [max_pos][64] tables in the model dtype (Q3)
  int kv_capacity;      // upper bound on keys per query (sizes the score buffer)
  float scale;
};
// prefill_tc: bf16 MHA prefill (q_len > 1) runs on the tensor-core sweep (attention_prefill_tc_kernel) rather than attention_item
int launch_attention(const AttnArgs& a, int dtype, cudaStream_t st, bool pdl, bool prefill_tc);

// ---- output_attentions / output_hidden_states (probe.cu) ----------------------------------------
// Decode window (both structs): ctrl != nullptr -> the step is ctrl->cur_len - n0, written to out + (step - first_step) * step_bytes
// when it lies in [first_step, first_step + n_steps), nothing otherwise or once ctrl->active is 0.  ctrl == nullptr: out as given.
struct AttnProbeArgs {
  const void* q; int64_t ldq; int q_col0;          // row b*q_len + j, head h at columns q_col0 + h*64 (before RoPE and scaling)
  const void* kcache; int64_t kv_b_stride, kv_h_stride;  // K rows [..][64], swizzled (kv_swz)
  int kv_b_div;                                    // row b reads K rows and key mask of batch index b / kv_b_div (AttnArgs)
  const int* key_mask; int mask_len, mask_ld;      // keys t < mask_len with key_mask[b*mask_ld+t] == 0 are masked
  int B, nh, nkv, q_len;
  int cross;                                       // 1: kv_len keys, no causal mask
  int kv_len, pos0;                                // ctrl == nullptr: keys per row, position of query row 0 (self: keys <= pos)
  int kv_cap;                                      // upper bound on keys per row (sizes shared memory)
  int rope; const void* rope_cos; const void* rope_sin;
  float scale;
  void* out; int64_t out_b, out_h, out_q;          // element strides of [B][nh][q_len][keys]; keys contiguous
  const Ctrl* ctrl; int n0, prefix, first_step, n_steps; int64_t step_bytes;  // decode: position = prefix + cur_len - 1
};
int launch_attention_probs(const AttnProbeArgs& a, int dtype, cudaStream_t st);
struct ProbeRowsArgs {
  const void* x; int rows, H;                      // [rows][H]
  const float* ln_w; const float* ln_b; float eps; // nullptr: copy; else the LayerNorm of each row
  int q_len; int64_t out_b;                        // row r = b*q_len + j goes to out + b*out_b + j*H
  void* out;
  const Ctrl* ctrl; int n0, first_step, n_steps; int64_t step_bytes;
};
int launch_probe_rows(const ProbeRowsArgs& a, int dtype, cudaStream_t st);
// return_token_timestamps (ptts_generate_set_alignment): one layer's share of the alignment row of a decode step.  The step's
// query is column c = ctrl->cur_len - 1; it writes row c - n0 - first_row of out ([n_rows][B][key_len] fp32) when that lies in
// [0, n_rows), nothing otherwise or once ctrl->active is 0.
struct AlignProbeArgs {
  const void* q; int64_t ldq; int q_col0;          // as AttnProbeArgs (decode: one query row per batch row)
  const void* kcache; int64_t kv_b_stride, kv_h_stride; int kv_b_div;
  const int* key_mask; int mask_ld;                // key t with key_mask[(b / kv_b_div) * mask_ld + t] == 0 gets weight 0
  int B, nh, nkv;
  int key0, key_len;                               // the transcript keys [key0, key0 + key_len)
  const int* heads; int n_heads; int layer;        // device [n_heads][2] (layer, head): the entries of `layer` are this launch's
  int layer_heads;                                 // how many entries belong to `layer`
  float weight;                                    // 1 / n_heads: the mean
  int accumulate;                                  // 0: the first layer with alignment heads stores, later layers add
  int rope; const void* rope_cos; const void* rope_sin;
  float scale;
  float* out;
  const Ctrl* ctrl; int n0, prefix, first_row, n_rows;
};
int launch_alignment_probe(const AlignProbeArgs& a, int dtype, cudaStream_t st);

// ---- token timestamps (align.cu) ----------------------------------------------------------------
// x [B][T][P] fp32 -> y (the width-7 median along frames of each utterance's first n_frames[b] rows), then per utterance the DTW
// of -y over its unmasked keys and frames; jumps [B][P] = the first frame of each key on the path (-1 for a masked key).
// trace: B * (P + 1) * (T + 1) bytes of scratch.
int launch_align_dtw(const float* x, int B, int T, int P, const int* n_frames, const int* key_mask, float* y, unsigned char* trace,
                     int* jumps, cudaStream_t st);

// ---- embedding (embed.cu) -----------------------------------------------------------------------
struct EmbedArgs {
  const void* tables;  // [K][V+1][H]
  const void* pos;     // [max_pos][H] or nullptr (rope)
  const void* prefix;  // [B][P][H] prompt hidden states or nullptr
  const int* ids;      // [B*K] current (delay-masked) input ids (decode)
  const int64_t* hist; int64_t hist_ld;  // prefill: [B*K][hist_ld] history whose first n_cols columns are the (delayed) input
  void* x;             // [B*(P+n_cols) or B][H]
  const Ctrl* ctrl;
  int B, K, V1, H, P;  // P = prefix rows per batch in THIS call (0 at decode)
  int n_cols;          // code columns per batch row after the prefix (1 at decode)
  int pos_from_ctrl, pos0, prefix_len;  // decode: position = prefix_len + cur_len - 1 - row_shift(shift, b)
  const int* shift;    // decode: per-row position offsets of a ragged continuation (SampleArgs::shift), or nullptr
};
int launch_embed(const EmbedArgs& a, int dtype, cudaStream_t st, bool pdl);

// ---- sampling / generation state (sample.cu) ----------------------------------------------------
struct SampleArgs {
  const float* logits; float* scores;  // [BK][V]
  int64_t* raw_ids; int64_t raw_ld;
  int* cur_ids; int* eos_seen; int* unfinished; int* first_unf;  // first_unf [2][B]
  Ctrl* ctrl;
  const ptts_gen_params* gen;  // device copy
  int64_t* prefix_cells;       // [B*K][K-1] pattern cells past a multi-column input (nullptr: the session takes the BOS column only)
  // [B] ragged continuation (ptts_generate_begin_ids2): row b's input is shift[b] columns shorter than the longest, and every
  // column it reads or writes is the batch's cur_len - shift[b] (its own, starting at 0); nullptr: all rows share cur_len
  int* shift;
  int B, K, V;
  int bos, pad, eos;
};
// generate()'s per-step outputs (ptts_generate_set_outputs): slot s of row r lives at ptr + (s - first_step) * step_stride + r * V
struct SampleOut {
  float* logits; float* scores;  // either may be nullptr
  int first_step, n_steps;       // the window of steps (step = cur_len - input_len) that are recorded
  int64_t step_stride;           // floats between consecutive slots
};
// ext != nullptr: the sampler with the ptts_sampling_ext stages (the caller passes it while one is active, or all off while out is
// set); out != nullptr (needs ext): that sampler also records the raw logits and the processed scores of the steps in its window
// lext: the ptts_logits_ext stages (needs ext; nullptr = all off)
// slot_key (needs ext and a.shift): slot mode (ptts_generate_set_slots2), with the per-row Philox keys [B] and slot_max_len, the
// per-row length limits [B], on the device
int launch_sample(const SampleArgs& a, const int64_t* forced, cudaStream_t st, bool pdl, const ptts_sampling_ext* ext = nullptr,
                  const SampleOut* out = nullptr, const ptts_logits_ext* lext = nullptr, const int* slot_key = nullptr,
                  const int* slot_max_len = nullptr);
// every ptts_logits_ext stage off
constexpr ptts_logits_ext kLogitsExtOff = {nullptr, nullptr, nullptr, 0, -1, -1, 0, nullptr, 0, nullptr, nullptr, 1, 0};
// the fused step kernels' sampling phase over n_ctas CTAs (passes of up to three rows per CTA), as a kernel of its own; no EXT
int launch_sample_phase(const SampleArgs& a, int n_ctas, cudaStream_t st);
// ids == nullptr: the BOS column (n0 = 1); otherwise the BOS-led [B*K][n0] input the generation continues from.  lens (with
// a.shift): row b's input is its first lens[b] columns (in [1, n0]); the kernel writes a.shift[b] = n0 - lens[b]
int launch_generate_begin(const SampleArgs& a, const int64_t* ids, int n0, int max_length, const int* lens, cudaStream_t st);
int launch_delay_build(const int64_t* ids, int BK, int seq, int K, int64_t bos, int64_t pad, int L, int64_t* mask, cudaStream_t st);
int launch_delay_apply(const int64_t* ids, int BK, int seq, int64_t ld_ids, const int64_t* mask, int64_t ld_mask, int64_t* out, cudaStream_t st);
int launch_logits_processor(const int64_t* ids, int BK, int seq, int64_t ld_ids, float* scores, int V, int64_t eos, int K, int64_t* first_unf, cudaStream_t st);
int launch_mask_convert(const int64_t* src, int n, int* dst, cudaStream_t st);  // int64 0/1 -> int32; src==nullptr -> ones
int launch_cross_kv_relayout(const void* src, void* dst, int B, int S, int nckv, int dtype, cudaStream_t st);
// dst row r = src row row0 + r * row_step - row_shift(shift, r)
int launch_gather_rows(const void* src, int64_t ld_src, int64_t row0, int64_t row_step, const int* shift, void* dst, int rows, int cols,
                       int dtype, cudaStream_t st);

// ---- continuous batching (rows.cu) --------------------------------------------------------------
// ptts_session_import_rows: row src_row[p] of the source workspace -> slot dst_row[p] of the destination, over the row_regions
// lists of both sessions (same config, P and S: the lists match entry for entry)
constexpr int kMaxImportRows = 32;   // row pairs per launch
struct RowImportArgs {
  const char* src_ws; char* dst_ws;
  const Ctrl* src_ctrl; const Ctrl* dst_ctrl;   // the history's length, and each side's first_unf parity
  RowRegion src[kMaxRowRegions], dst[kMaxRowRegions];
  int n_regions, K;   // K: codebooks (first_unf holds row indices b * K + k)
  int src_row[kMaxImportRows], dst_row[kMaxImportRows];
};
int launch_import_rows(const RowImportArgs& a, int n_pairs, cudaStream_t st);
// slot mode (ptts_generate_set_slots2): the host arrays row_shift / row_key / row_max_len [B] into the workspace's shift / key /
// max_len, then the new cur_len, active = 1 and the sampler's counters cleared
constexpr int kMaxSlotRows = 256;    // rows per launch
int launch_set_slots(Ctrl* ctrl, int cur_len, int* shift, int* key, int* max_len, const int* row_shift, const int* row_key,
                     const int* row_max_len, int B, cudaStream_t st);

// ---- teacher-forced scoring (score.cu) ----------------------------------------------------------
struct ScoreArgs {
  const int64_t* labels;   // [B][T][K] int64, -100 = ignored (nullptr: logits only, no NLL)
  const int64_t* dec_ids;  // [B*K][T] int64: the decoder input (a cell whose input id is eos is not counted)
  float* token_nll;        // [B][T][K] f32: logsumexp - logit[label], 0 where the cell is not counted
  const float* c1; const float* c2;  // fused kernel: the heads' folded-LayerNorm vectors [K*V]
  int M, B, T, K, V, H;    // M = B*T label rows
  int bos, eos;
};
bool score_fused_supported(int H, int V);
// bf16: x = the decoder output [B][P+T][H]; gathers the label rows into xs_scratch [M][H] (+ LayerNorm stats), then the fused
// heads + cross-entropy kernel over heads_rm (row-major folded heads [K*V][H])
int launch_score_fused(const ScoreArgs& a, const void* x, int P, float eps, void* xs_scratch, float* stats_scratch,
                       const void* heads_rm, cudaStream_t st);
// unfused, frame t: the heads GEMM's f32 logits [B*K][V] -> token_nll (labels != nullptr) and logits_out [B*K][T][V] (if set)
int launch_score_rows(const ScoreArgs& a, const float* logits, int t, float* logits_out, cudaStream_t st);
// out [K][2] f32: per codebook, the sum of token_nll over counted cells and their count
int launch_score_reduce(const ScoreArgs& a, float* out, cudaStream_t st);

}  // namespace ptts
