/*
 * ptts_b200.h -- C ABI of the H100-native (sm_90a) Parler-TTS generation path.
 *
 * Drop-in boundary: the reference (huggingface/parler-tts) has NO native layer; its hot path is
 * Python calling stock PyTorch ops.  Each entry point below names the reference interface it
 * replaces (file:line under the reference repo).  The Python shim in parler_tts_b200/ mirrors the
 * reference's public classes and calls these functions through ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no torch / C++ types.
 *   - every function returns 0 on success, non-zero on error; ptts_last_error() gives the message
 *     (thread-local).  The Python shim raises ValueError (PTTS_EINVAL) or RuntimeError (others),
 *     matching the reference's ValueError-on-contract-violation behaviour
 *     (e.g. dac_wrapper/modeling_dac.py:135-136, modeling_parler_tts.py:3471-3475).
 *   - the library never allocates caller-visible device memory: weights blob and workspace are
 *     caller-allocated (torch tensors), sized by the *_bytes() queries.
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream);
 *     `device` pointers are raw CUDA device pointers on the current device of the calling thread.
 *   - dtype codes: 0 = bf16, 1 = f32, 2 = int64, 3 = int32.
 */
#ifndef PTTS_B200_H
#define PTTS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PTTS_OK 0
#define PTTS_EINVAL 1   /* contract violation -> ValueError */
#define PTTS_ECUDA 2    /* CUDA runtime error -> RuntimeError */
#define PTTS_ESTATE 3   /* wrong call order   -> RuntimeError */

#define PTTS_BF16 0
#define PTTS_F32 1
#define PTTS_I64 2
#define PTTS_I32 3

#define PTTS_HEAD_DIM 64

/* ParlerTTSDecoderConfig fields the path needs (configuration_parler_tts.py:107-172). */
typedef struct ptts_decoder_config {
  int32_t hidden_size;
  int32_t num_layers;
  int32_t num_heads;
  int32_t num_kv_heads;        /* self-attention KV heads (GQA, :948) */
  int32_t num_cross_kv_heads;  /* cross-attention KV heads (:970) */
  int32_t ffn_dim;
  int32_t vocab_size;          /* lm-head rows; embedding tables have vocab_size+1 rows (:1353) */
  int32_t num_codebooks;
  int32_t max_positions;
  int32_t rope;                /* rope_embeddings (:130); 0 -> sinusoidal table added to embeds */
  int32_t activation;          /* 0 gelu(erf), 1 relu, 2 silu, 3 gelu(tanh) */
  int32_t dtype;               /* PTTS_BF16 or PTTS_F32: model dtype (weights, activations, KV) */
  int32_t bos_token_id, pad_token_id, eos_token_id;
  float rope_theta;
  float layer_norm_eps;
} ptts_decoder_config;

/* Generation knobs (HF GenerationConfig subset used by generate(), modeling_parler_tts.py:3395-3552). */
typedef struct ptts_gen_params {
  int32_t max_length;      /* total decoder length incl. BOS column */
  int32_t min_new_tokens;
  int32_t do_sample;       /* 0 = greedy argmax */
  int32_t top_k;           /* 0 = off */
  float top_p;             /* >= 1 = off */
  float temperature;       /* 1 = off */
  uint64_t seed;           /* Philox key; substream = (row_base + row, step) */
  int32_t suppress_special; /* bench aid: mask ids >= codebook_size (never set by generate()) */
  int32_t codebook_size;
  int32_t row_base;        /* global index of this session's first row (= first utterance * num_codebooks): with a batch
                            * sharded over GPUs every shard passes its own offset, so the draws of an utterance do not
                            * depend on the number of shards (SURVEY 8e) */
  int32_t input_len;       /* n0: columns of the BOS-led decoder input the generation continues from (0 means 1, the BOS
                            * column alone).  MinNewTokens skips these columns.  ptts_generate_begin_ids sets it. */
} ptts_gen_params;

/* The further processors of transformers' _get_logits_processor, in its order: NoRepeatNGram before the EOS masks' processors,
 * then, when sampling, MinP, Typical, Epsilon and Eta after top-p.  All zero except typical_p = 1 is off. */
typedef struct ptts_sampling_ext {
  int32_t no_repeat_ngram_size; /* 0 = off; greedy and sampling: bans the next id of every earlier n-gram that repeats the
                                 * row's last n-1 ids */
  float min_p;                  /* [0, 1]: remove p < min_p * p_max (sampling only; 0 = off) */
  float typical_p;              /* (0, 1]: locally typical mass (sampling only; 1 = off) */
  float epsilon_cutoff;         /* [0, 1): remove p < epsilon (sampling only; 0 = off) */
  float eta_cutoff;             /* [0, 1): remove p < min(eta, sqrt(eta) exp(-entropy)) (sampling only; 0 = off) */
} ptts_sampling_ext;

/* The remaining processors of transformers' _get_logits_processor (modeling_parler_tts.py:3540-3547), greedy and sampling.  On
 * each step's fp32 row, with cur_len = the column being drawn (the history's length), they run in transformers' order:
 *   SequenceBias, [NoRepeatNGram], [MinNewTokens], ForcedBOS, ForcedEOS, InfNanRemove, ExponentialDecayLengthPenalty, Suppress,
 *   SuppressAtBegin, [ParlerTTSLogitsProcessor], [temperature .. eta], LogitNormalization.
 * Every table is caller-owned device memory that must stay valid while the generation runs; a NULL table (or a negative id) is
 * that stage off.  All off = every pointer NULL, both ids -1, both flags 0. */
#define PTTS_SEQ_BIAS_MAX 64       /* multi-id sequences of sequence_bias */
#define PTTS_SEQ_BIAS_MAX_LEN 16   /* ids per sequence */
typedef struct ptts_logits_ext {
  /* SequenceBiasLogitsProcessor: row[i] += (0 + bias1[i]) + the bias of every sequence in `seq` whose last id is i and whose
   * other ids equal the last len-1 history ids, added in table order (sequences longer than cur_len are skipped) */
  const float* bias1;           /* [V] the single-id biases (0 where none), or NULL */
  const int32_t* seq;           /* [n_seq][1 + PTTS_SEQ_BIAS_MAX_LEN]: len, then the len ids (oldest first) */
  const float* seq_bias;        /* [n_seq] */
  int32_t n_seq;                /* [0, PTTS_SEQ_BIAS_MAX] */
  int32_t forced_bos_token_id;  /* ForcedBOSTokenLogitsProcessor: at cur_len == 1, every id -inf but this one, which gets 0; -1 = off */
  int32_t forced_eos_token_id;  /* ForcedEOSTokenLogitsProcessor: the same at cur_len == max_length - 1; -1 = off */
  int32_t remove_invalid_values; /* InfNanRemoveLogitsProcessor: NaN -> 0, +-inf -> +-FLT_MAX; 0 = off */
  /* ExponentialDecayLengthPenalty: at cur_len > decay_start (= start + n0), row[eos] += |row[eos]| * decay[cur_len], where the
   * caller fills decay[c] = (float)(factor^(c - decay_start) - 1) in double precision; the other ids get + 0 */
  const float* decay;           /* [max_length], or NULL */
  int32_t decay_start;
  const uint32_t* suppress;     /* SuppressTokensLogitsProcessor: bitmap of ids, [ceil(V / 32)] words, bit i % 32 of word i / 32 */
  const uint32_t* begin_suppress; /* SuppressTokensAtBeginLogitsProcessor: bitmap, applied at cur_len == begin_index only */
  int32_t begin_index;          /* n0, or 2 when n0 == 1 and forced_bos_token_id is set (_get_logits_processor) */
  int32_t renormalize_logits;   /* LogitNormalization: the recorded scores are log_softmax of the final row; the token is drawn
                                 * from the same distribution as without it (softmax(log_softmax(x)) = softmax(x)), and greedy's
                                 * argmax is taken before the normalization; 0 = off */
} ptts_logits_ext;

/* Tensor ids for ptts_decoder_pack(). `index` = layer (per-layer tensors) or codebook (EMBED/LM_HEAD). */
enum {
  PTTS_T_EMBED_TOKENS = 0, /* [vocab+1, H]  decoder.model.decoder.embed_tokens.N.weight (:1354) */
  PTTS_T_POS_TABLE = 1,    /* [max_pos, H]  embed_positions.weights (:1360), absent when rope */
  PTTS_T_LN1_W = 2, PTTS_T_LN1_B = 3,      /* self_attn_layer_norm (:961) */
  PTTS_T_SELF_Q = 4, PTTS_T_SELF_K = 5, PTTS_T_SELF_V = 6, PTTS_T_SELF_O = 7,    /* :481-484 */
  PTTS_T_LN2_W = 8, PTTS_T_LN2_B = 9,      /* encoder_attn_layer_norm (:978) */
  PTTS_T_CROSS_Q = 10, PTTS_T_CROSS_K = 11, PTTS_T_CROSS_V = 12, PTTS_T_CROSS_O = 13,
  PTTS_T_LN3_W = 14, PTTS_T_LN3_B = 15,    /* final_layer_norm (:981) */
  PTTS_T_FC1 = 16, PTTS_T_FC2 = 17,        /* :979-980 */
  PTTS_T_FINAL_LN_W = 18, PTTS_T_FINAL_LN_B = 19, /* decoder.layer_norm (:1373) */
  PTTS_T_LM_HEAD = 20,     /* [vocab, H] decoder.lm_heads.N.weight (:1838) */
  PTTS_T_ROPE_COS = 21,    /* [max_pos, 64] cos table, fp32 -> model dtype as the reference does (:394-406, :1534) */
  PTTS_T_ROPE_SIN = 22,    /* [max_pos, 64] sin table (only when rope != 0) */
  PTTS_T_COUNT = 23
};

const char* ptts_last_error(void);
int ptts_version(void);

/* ---- decoder: weights --------------------------------------------------------------------- */
/* Size of the packed weight blob (device bytes) for this config. */
int ptts_decoder_blob_bytes(const ptts_decoder_config* cfg, int64_t* out_bytes);
/* Repack one reference-layout tensor (row-major [rows, cols], dtype src_dtype, device memory) into
 * the blob: GEMM matrices go to MMA-fragment order (bf16) / row-major (f32); q,k,v are fused into one
 * matrix; LayerNorm parameters are kept in f32.  Replaces nothing in the reference (load-time only). */
int ptts_decoder_pack(const ptts_decoder_config* cfg, void* blob, int32_t tensor_id, int32_t index,
                      const void* src, int32_t src_dtype, int64_t rows, int64_t cols, void* stream);

/* Call once after every tensor has been packed (bf16 model dtype): folds each LayerNorm's affine part into the
 * linear layer that follows it (W' = gamma*W, c1 = rowsum(W'), c2 = W*beta), so that the run-time GEMM consumes the
 * raw residual stream and only needs per-row (mean, rstd).  No-op for f32. */
int ptts_decoder_finalize(const ptts_decoder_config* cfg, void* blob, void* stream);

/* ---- decoder: generation session ----------------------------------------------------------- */
/* Workspace bytes for a batch of B utterances, prompt prefix length P, encoder length S and a
 * self-attention cache of max_cache_len positions (>= P + max_length - 1). */
int ptts_workspace_bytes(const ptts_decoder_config* cfg, int32_t B, int32_t P, int32_t S,
                         int32_t max_cache_len, int64_t* out_bytes);

/* Same, for a session that may continue from up to max_input_len decoder input columns (ptts_generate_begin_ids): the prefill
 * activations are sized for B * (P + max_input_len) rows.  max_input_len = 1 gives exactly ptts_workspace_bytes. */
int ptts_workspace_bytes2(const ptts_decoder_config* cfg, int32_t B, int32_t P, int32_t S, int32_t max_cache_len,
                          int32_t max_input_len, int64_t* out_bytes);

/* Same, for a session whose B rows are B / takes descriptions with `takes` consecutive takes each (generate(num_return_sequences=
 * takes), modeling_parler_tts.py:3556): row b reads the cross-attention K/V and encoder mask of description b / takes, so the
 * workspace holds those for B / takes descriptions only.  takes must divide B (PTTS_EINVAL otherwise); takes = 1 gives exactly
 * ptts_workspace_bytes2. */
int ptts_workspace_bytes3(const ptts_decoder_config* cfg, int32_t B, int32_t P, int32_t S, int32_t max_cache_len,
                          int32_t max_input_len, int32_t takes, int64_t* out_bytes);

typedef struct ptts_session ptts_session; /* host-side object: pointers into blob/workspace + CUDA graphs */

int ptts_session_create(const ptts_decoder_config* cfg, const void* blob, void* workspace,
                        int64_t workspace_bytes, int32_t B, int32_t P, int32_t S, int32_t max_cache_len,
                        ptts_session** out);
/* Same, with the max_input_len of ptts_workspace_bytes2 (= ptts_session_create when 1). */
int ptts_session_create2(const ptts_decoder_config* cfg, const void* blob, void* workspace,
                         int64_t workspace_bytes, int32_t B, int32_t P, int32_t S, int32_t max_cache_len,
                         int32_t max_input_len, ptts_session** out);
/* Same, with the takes of ptts_workspace_bytes3 (= ptts_session_create2 when 1).  On such a session ptts_prefill and ptts_score
 * take enc_hidden [B / takes, S, H] and enc_mask [B / takes, S]: the cross-attention K/V are projected once per description and
 * shared by its takes in every decode path.  Everything else (prompt prefix, decoder input, outputs, probes) has B rows. */
int ptts_session_create3(const ptts_decoder_config* cfg, const void* blob, void* workspace,
                         int64_t workspace_bytes, int32_t B, int32_t P, int32_t S, int32_t max_cache_len,
                         int32_t max_input_len, int32_t takes, ptts_session** out);
int ptts_session_destroy(ptts_session* s);

/* Start a generate() call: reset per-call state (ids history = BOS column, processor state,
 * unfinished flags, delay-pattern parameters).  Replaces generate() steps 5-9
 * (modeling_parler_tts.py:3449-3552), build_delay_pattern_mask (:3523) and the
 * ParlerTTSLogitsProcessor constructor (logits_processors.py:23-42). */
int ptts_generate_begin(ptts_session* s, const ptts_gen_params* gen, void* stream);

/* Start a generate() call that continues from audio codes (decoder_input_ids, modeling_parler_tts.py:2988-3024, :3523).
 *   input_ids [B*K, n0] int64 device, BOS-led (the caller prepends the BOS column, :3012-3024), ids in [0, vocab_size];
 *             NULL with n0 == 1 is the BOS column (= ptts_generate_begin).  1 <= n0 <= max_input_len, n0 < gen->max_length.
 * On the device, without a host sync: the delayed input (the first n0 columns of build_delay_pattern_mask(input_ids, bos, pad,
 * max_length), :214-276) becomes the history, the K-1 pattern cells past it are kept for the next-input override (:2909),
 * cur_len = n0, and the processor state sees the EOS ids inside the prefix.  ptts_prefill then runs the prompt prefix and the n0
 * columns in one pass (:3033-3044); gen->input_len is set to n0. */
int ptts_generate_begin_ids(ptts_session* s, const ptts_gen_params* gen, const int64_t* input_ids, int32_t n0, void* stream);

/* Same, for a batch whose rows continue from inputs of different lengths (ragged prefixes).
 *   input_lens [B] int32 device, or NULL (= ptts_generate_begin_ids): row b's input is the first n0_b = input_lens[b] columns of
 *              its input_ids row, 1 <= n0_b <= n0 (the columns past it are never read).  Checked with one host sync.  With
 *              n0 == 1 every length is 1: the call is ptts_generate_begin_ids (any session takes it).
 * Row b then computes exactly what it would as a batch of its own, continuing from its n0_b columns with max_length
 * gen->max_length - (n0 - n0_b): its history, cache slots and positions start at 0 as they would alone, and every decode step,
 * sampler stage and Philox draw uses its own column cur_len - (n0 - n0_b).  All rows reach their limit at the same step.  The
 * probe windows (ptts_generate_set_probes, ptts_generate_set_alignment) are refused while such a call runs. */
int ptts_generate_begin_ids2(ptts_session* s, const ptts_gen_params* gen, const int64_t* input_ids, int32_t n0, const int32_t* input_lens,
                             void* stream);

/* Step 0 (prefill): prompt prefix + the n0 delayed input columns (the BOS column unless the call began with
 * ptts_generate_begin_ids) through the decoder, cross-attention K/V projected once,
 * self-attention cache filled at positions [0, P + n0).  Leaves f32 logits [B*K, V] in the workspace.
 * Replaces ParlerTTSForCausalLM.forward at step 0 (:1865-1974, :1392-1655, :872-889).
 *   prompt_hidden [B, P, H] model dtype (may be NULL when P == 0)   (:3099-3134 output)
 *   prompt_mask   [B, P] int64 or NULL                              (prompt_attention_mask)
 *   enc_hidden    [B, S, H] model dtype, already multiplied by the mask (:3092-3093)
 *   enc_mask      [B, S] int64 or NULL                              (attention_mask)            */
int ptts_prefill(ptts_session* s, const void* prompt_hidden, const int64_t* prompt_mask,
                 const void* enc_hidden, const int64_t* enc_mask, void* stream);

/* ---- teacher-forced scoring ---------------------------------------------------------------- */
/* The fused scoring kernel reads the K lm heads row-major ([K*V][H] bf16, LayerNorm folded as in the blob).  The blob keeps them
 * in mma fragment order only, so the copy lives in a separate caller-owned buffer of ptts_lm_heads_rowmajor_bytes bytes, filled
 * by ptts_lm_heads_rowmajor_pack after ptts_decoder_finalize.  bf16 models only (PTTS_EINVAL otherwise). */
int ptts_lm_heads_rowmajor_bytes(const ptts_decoder_config* cfg, int64_t* out_bytes);
int ptts_lm_heads_rowmajor_pack(const ptts_decoder_config* cfg, const void* blob, void* heads_rm, void* stream);

/* The teacher-forced forward with labels (ParlerTTSForConditionalGeneration.forward, :2695-2880; loss :1922-1974) on a session
 * created with max_input_len >= T: the prompt prefix and the T decoder input columns go through the decoder in one prefill pass,
 * then the K lm heads run over the T label positions of every utterance.
 *   prompt_hidden, prompt_mask, enc_hidden, enc_mask   as for ptts_prefill
 *   dec_ids   [B*K, T] int64 in [0, vocab_size]: the decoder input AS GIVEN (already delayed / shifted; no delay is applied)
 *   labels    [B, T, K] int64 in {-100} u [0, vocab_size), or NULL (logits only).  As in the reference, a BOS label counts as
 *             -100, and a cell (b, t, k) counts iff labels != -100 and dec_ids[b*K + k][t] != eos.
 *   heads_rm  the row-major heads (ptts_lm_heads_rowmajor_pack): required by the fused bf16 path, unused otherwise
 *   out_token_nll      [B, T, K] f32: logsumexp(logits) - logits[label] per counted cell, 0 elsewhere (needs labels)
 *   out_logits         NULL, or [B*K, T, V] f32: the logits (the unfused route: the decoder's heads GEMM one frame at a time)
 *   out_codebook_sums  NULL, or [K][2] f32: per codebook the sum of out_token_nll over counted cells and their count
 * bf16 without out_logits runs the fused heads + cross-entropy kernel (the logits never reach memory); f32 models and calls that
 * want the logits take the unfused route.  The session's caches and history are overwritten: a generation on it starts again
 * with ptts_generate_begin*. */
int ptts_score(ptts_session* s, const void* prompt_hidden, const int64_t* prompt_mask, const void* enc_hidden,
               const int64_t* enc_mask, const int64_t* dec_ids, const int64_t* labels, int32_t T, const void* heads_rm,
               float* out_token_nll, float* out_logits, float* out_codebook_sums, void* stream);

/* One cached decode step for the ids currently staged in the workspace (the delay-masked last
 * column).  Leaves f32 logits [B*K, V] in the workspace.  Replaces prepare_inputs_for_generation
 * (:2882-2986) + ParlerTTSForCausalLM.forward with q_len == 1. */
int ptts_decode_forward(ptts_session* s, void* stream);

/* logits -> next token for every row, on device: MinNewTokens, ParlerTTSLogitsProcessor
 * (logits_processors.py:44-53), temperature/top-k/top-p, softmax + sampling or argmax, finished-row
 * padding, history append, EOS/max-length stopping, delay-mask override of the next input.
 * Replaces one iteration of GenerationMixin._sample (transformers 4.46.1) + :2909.
 * forced_tokens: NULL, or [B*K] int64 device tokens that replace the drawn ones (teacher forcing). */
int ptts_sample(ptts_session* s, const int64_t* forced_tokens, void* stream);

/* n_steps x (ptts_decode_forward + ptts_sample), replayed from a CUDA graph, no host sync.
 * Steps after every row finished are device-side no-ops. */
int ptts_decode_steps(ptts_session* s, int32_t n_steps, void* stream);

/* The processors of ptts_sampling_ext for the generation begun last (ptts_generate_begin* resets them to off; NULL = off).
 * Out-of-range values give PTTS_EINVAL.  While any is active (no_repeat_ngram_size > 0, or a warper with do_sample),
 * ptts_sample runs a sampler that applies them, and ptts_decode_steps runs every token as the decoder step without its
 * sampling phase followed by that sampler: one launch pair per token instead of the step kernel's many tokens per launch.
 * A row left with no candidate gets token 0 (the reference's torch.multinomial raises there). */
int ptts_generate_set_sampling_ext(ptts_session* s, const ptts_sampling_ext* ext);

/* The processors of ptts_logits_ext for the generation begun last (ptts_generate_begin* resets them to off; NULL = off).  The
 * struct is copied; the tables it points to are read by every step.  PTTS_EINVAL for n_seq outside [0, PTTS_SEQ_BIAS_MAX], n_seq > 0
 * with a NULL seq or seq_bias, a forced id outside [-1, vocab_size), decay_start < 0 or begin_index < 1.  The sequence table is not
 * read on the host: the sampler skips a sequence whose len is outside [2, PTTS_SEQ_BIAS_MAX_LEN], and ids are only compared, so
 * one outside [0, V) never matches (the Python shim rejects both first).  While any stage is active, ptts_sample and
 * ptts_decode_steps take the split path of ptts_generate_set_sampling_ext. */
int ptts_generate_set_logits_ext(ptts_session* s, const ptts_logits_ext* ext);

/* generate()'s output_logits / output_scores for the generation begun last: the sampler records, for every step (step =
 * cur_len - n0, the column it draws minus the decoder input's columns) inside [first_step, first_step + n_steps), the raw f32
 * logits row it reads and the processed scores row the token is drawn from (after every processor and warper; removed ids are
 * -inf).  Buffers are caller-owned device memory; slot s of row r is at ptr + (s - first_step) * step_stride + r * V floats, so a
 * shard passes a pointer to its first row inside a whole-batch buffer.  Either pointer may be NULL; both NULL = off, which
 * ptts_generate_begin* restores.  PTTS_EINVAL for first_step < 0, n_steps < 0 or step_stride < B*K*V.  May be called between
 * ptts_decode_steps calls to move the window.  While set, ptts_sample and every token of ptts_decode_steps run the EXT sampler
 * (the split path of ptts_generate_set_sampling_ext; the step kernels' own sampling phase is not used), and the multi-kernel
 * path's graph is captured again when the window moves.  Steps after the generation stopped write nothing. */
int ptts_generate_set_outputs(ptts_session* s, float* logits, float* scores, int32_t first_step, int32_t n_steps,
                              int64_t step_stride);

/* output_attentions / output_hidden_states: the decoder passes write, for every step inside [first_step, first_step + n_steps)
 * (step 0 = the prefill of ptts_prefill or ptts_score, with q = P + n0 rows; step t >= 1 = the decode step whose token is column
 * n0 + t, q = 1), into caller-owned device buffers in the model dtype.  Slot s (= step - first_step) starts at ptr + s * *_step
 * elements and holds, for q rows per batch row:
 *   self_attn  [B][L][nh][q][self_ld]   the self-attention weights of T_kv = P + n0 + step keys (the prefill: P + n0) in the
 *                                       first T_kv elements of each row; self_ld >= the longest T_kv of the window
 *   cross_attn [B][L][nh][q][S]         the cross-attention weights
 *   hidden     [B][L + 1][q][H]         the residual stream after the embedding and after layers 0 .. L-2, then the final
 *                                       LayerNorm of the last layer's output
 * Batch rows are outermost, so a shard passes pointers to its first row inside whole-batch buffers (the step strides then span
 * the whole batch).
 * The weights follow the reference's eager attention (dtype scores, fp32 softmax, finfo.min mask), from the q and K the session's
 * own attention reads; the tokens do not depend on them.  Any pointer may be NULL; all NULL = off, which ptts_generate_begin*
 * restores.  While a window is set, ptts_decode_steps and ptts_decode_forward run the multi-kernel path (the step kernels hold
 * no per-layer state to write out), whose graph is captured again whenever the window moves; ptts_session_fused still reports the
 * path the session uses without one.  PTTS_EINVAL for a negative window, self_ld below the window's longest row or strides below
 * one slot. */
int ptts_generate_set_probes(ptts_session* s, void* self_attn, void* cross_attn, void* hidden, int32_t first_step, int32_t n_steps,
                             int64_t self_ld, int64_t self_step, int64_t cross_step, int64_t hidden_step);

/* return_token_timestamps: each decode step writes the transcript alignment of its query into a caller-owned fp32 buffer.  The
 * step whose input is column c (its query; the prefill writes nothing) writes row r = c - n0 when r lies in [first_step,
 * first_step + n_steps), at out + ((r - first_step) * B + b) * key_len floats: the mean over the n_heads listed heads (heads:
 * device int32 [n_heads][2] = (layer, head)) of each head's attention weights over keys [key0, key0 + key_len), renormalized
 * over those keys (a key whose mask is 0 gets weight 0).  The keys are the self-attention prompt prefix of a session with P > 0,
 * else its cross-attention keys.  Scores follow ptts_generate_set_probes' eager definition from the same q and K; the kernel
 * reads only the key_len transcript keys of each listed head.  out NULL = off, which ptts_generate_begin* restores; while set,
 * decode steps run the multi-kernel path as with probes.  The head list is copied to the host once here (a synchronous copy).
 * PTTS_EINVAL for an empty list, a head outside the model or listed twice, keys outside the session or a negative window. */
int ptts_generate_set_alignment(ptts_session* s, const int32_t* heads, int32_t n_heads, int32_t key0, int32_t key_len, float* out,
                                int32_t first_step, int32_t n_steps);

/* Token timestamps from alignments [B][T][P] fp32 (openai-whisper's recipe as transformers' generation_whisper states it): per
 * utterance b, the median of width 7 along its first n_frames[b] frames (reflect padding; <= 3 frames are left as they are)
 * into filtered [B][T][P], then the DTW of -filtered over those frames and the keys with key_mask[b][p] != 0 (masked keys are
 * removed, not given a cost; key_mask NULL = none masked), with _dynamic_time_warping's recurrence, fp32 sums and tie order
 * (diagonal, then previous key, then previous frame).  jumps [B][P] int32: the first frame of each key on the path, -1 for a
 * masked key, 0 for every key of an utterance without frames.  n_frames and key_mask are device int32 arrays; trace is
 * B * (P + 1) * (T + 1) bytes of device scratch.  Rows of filtered past n_frames[b] are not written. */
int ptts_align_dtw(const float* alignment, int32_t B, int32_t T, int32_t P, const int32_t* n_frames, const int32_t* key_mask,
                   float* filtered, uint8_t* trace, int32_t* jumps, void* stream);

/* ---- continuous batching ---------------------------------------------------------------------- */
/* Copy n request rows out of src into slots of dst: row src_rows[i] of src becomes row dst_rows[i] of dst (host int32 arrays; the
 * destination rows distinct).  src has run ptts_generate_begin (the BOS column), ptts_prefill and exactly one ptts_sample since, and
 * no decode step (PTTS_EINVAL otherwise: its cache holds positions [0, P + 1) and its history columns [0, 2) only then);
 * dst is prefilled, typically live in slot mode.  Both run the same model with the same config, P and S, takes = 1, the same
 * max_input_len class (1, or >= 2) and the same masks given at their prefills.  Every per-row region the decode path reads is
 * copied: the self K/V of positions [0, P + 1) of every layer and head, the cross K/V, the encoder and prompt masks, the history
 * columns [0, 2), the next input, the EOS and stopping state, the ParlerTTSLogitsProcessor state (into the parity
 * buffer dst's next step reads: keep dst's cur_len parity until then, see ptts_generate_set_slots) and the prefix cells.  One
 * kernel on `stream`, no host sync.  PTTS_ESTATE before either prefill; PTTS_EINVAL for sessions that do not match or rows out
 * of range. */
int ptts_session_import_rows(ptts_session* dst, const ptts_session* src, const int32_t* src_rows, const int32_t* dst_rows, int32_t n,
                             void* stream);

/* Slot mode: every row b is a request of its own that started from the BOS column, at its own column col_b = cur_len - row_shift[b]
 * (>= 1), with Philox key row_key[b] (its draws use substream row_key[b] * K + k, what row row_key[b] of a generate() call with
 * row_base 0 uses).  Each decode step then stops a row at col_b + 1 >= max_length or its EOS, masks EOS while col_b - 1 <
 * min_new_tokens and applies the delay pattern of max_length in the row's own column; the decode kernels put the row at position
 * P + col_b - 1.  Sets ctrl cur_len, reactivates a session that went inactive and clears the sampler's counters; row_shift and
 * row_key are host int32 [B] arrays, passed to the kernel by value (no host sync).  Call it again at every rebase.
 * Needs a prefilled session created with max_input_len >= 2 (it holds the per-row offsets), takes = 1, a generation begun from
 * the BOS column, no probe, alignment or per-step output window, and none of forced_eos_token_id, the decay penalty or
 * begin_suppress_tokens (they count from one batch column); every token then takes the split path's EXT sampler.  The caller
 * runs at most raw_ld - max(col_b) steps before the next call (ptts_session_raw_ids gives raw_ld), and keeps each row's
 * cur_len parity where it was when it imported rows.  Slot mode lasts until the next ptts_generate_begin*.
 * Same as ptts_generate_set_slots2 with row_max_length NULL. */
int ptts_generate_set_slots(ptts_session* s, int32_t cur_len, const int32_t* row_shift, const int32_t* row_key, void* stream);

/* ptts_generate_set_slots with a length limit per row: row b stops at col_b + 1 >= row_max_length[b] (or its EOS) and takes the
 * delay pattern of row_max_length[b] in its own column, what a generate() call with max_length = row_max_length[b] gives it.
 * row_max_length: host int32 [B], passed by value like the others, each in [max(2K - 1, 2), the generation's max_length]
 * (PTTS_EINVAL otherwise); NULL gives every row the generation's max_length.  The lower bound keeps a request's first column,
 * drawn before slot mode under the generation's max_length (ptts_sample of the session it is imported from), the one its own
 * limit gives: both limits are then on the same side of the delay pattern's 2K - 1 gate, and neither stops or pads column 1. */
int ptts_generate_set_slots2(ptts_session* s, int32_t cur_len, const int32_t* row_shift, const int32_t* row_key,
                             const int32_t* row_max_length, void* stream);

/* Device pointers into the workspace (valid for the session lifetime). */
int ptts_session_logits(ptts_session* s, float** out);          /* [B*K, V] f32, last step's raw logits */
int ptts_session_scores(ptts_session* s, float** out);          /* [B*K, V] f32, processed scores      */
int ptts_session_raw_ids(ptts_session* s, int64_t** out, int32_t* ld); /* [B*K, ld] raw (un-masked) history */
int ptts_session_state(ptts_session* s, int32_t** out);         /* int32[8]: {cur_len, n_unfinished, ...} */
int ptts_session_eos_seen(ptts_session* s, int32_t** out);      /* [B*K] int32: 1 + the column of each row's first EOS, 0 = none */
int ptts_session_launches(ptts_session* s, int64_t* out);       /* kernels launched through this session  */
/* After ptts_prefill: 0 = decode steps run the multi-kernel path (shape outside the fused kernel's range; a warning is printed
 * once), 1 = the fused persistent step kernel (one launch per token, step.cu), 2 = its cluster variant (step2.cu). */
int ptts_session_fused(ptts_session* s, int32_t* out);
/* Profiling aid: per-phase clock64() stamps of the fused step kernel into buf (device int64 [(8L+3)*8]); NULL = off. */
int ptts_session_set_profile(ptts_session* s, void* buf);

/* ---- stand-alone operators (same kernels, used by the Python mirrors and the tests) -------- */
/* build_delay_pattern_mask (:214-276): input_ids [B*K, seq] int64 -> pattern_mask [B*K, max_length]
 * int64 (the truncated input_ids the reference also returns is a slice the shim takes). */
int ptts_delay_build(const int64_t* input_ids, int32_t BK, int32_t seq_len, int32_t num_codebooks,
                     int64_t bos, int64_t pad, int32_t max_length, int64_t* pattern_mask, void* stream);
/* apply_delay_pattern_mask (:205-211): out = where(mask[:, :seq]==-1, ids, mask). */
int ptts_delay_apply(const int64_t* input_ids, int32_t BK, int32_t seq_len, int64_t ld_ids,
                     const int64_t* pattern_mask, int64_t ld_mask, int64_t* out, void* stream);
/* ParlerTTSLogitsProcessor.__call__ (logits_processors.py:44-53): scores [B*K, V] f32 in place;
 * first_unfinished [B] int64 is the processor's persistent state. */
int ptts_logits_processor(const int64_t* input_ids, int32_t BK, int32_t seq_len, int64_t ld_ids,
                          float* scores, int32_t V, int64_t eos, int32_t num_codebooks,
                          int64_t* first_unfinished, void* stream);
/* The fused step kernels' sampling phase (sample_all_rows_cta: each of n_ctas CTAs takes rows cta, cta + n_ctas, ..., one row
 * per pass while B*K <= n_ctas, otherwise passes of three) on the session's current logits, as a kernel of its own.  Test hook
 * for the three-row passes: it computes what ptts_sample computes (scores, the token at column cur_len and the per-row state)
 * but leaves cur_len where it is.  The per-row state it writes (unfinished, eos_seen, the next input) is the state after this
 * column, so a second launch at the same column, or a ptts_sample after it, repeats the result only while no row finished
 * there (drew EOS or reached max_length): such a row then gets PAD instead of its draw.  PTTS_ESTATE before ptts_prefill; PTTS_EINVAL for n_ctas < 1, vocab_size > 2304, or while a
 * ptts_sampling_ext stage or a ptts_generate_set_outputs window is active (the step kernels run neither). */
int ptts_op_sample_phase(ptts_session* s, int32_t n_ctas, void* stream);
/* y[M,N] = epi(LN?(x[M,K]) @ W^T): W taken from a packed blob slot (the whole fused matrix it belongs to).  Test hook for the
 * GEMM kernels.  path 0: the decode GEMM (launch_linear, every dtype); path 1: the wgmma prefill GEMM (launch_linear_tc) over
 * the matrix's row-major copy, with the same eligibility rule and the same blob lookup as the prefill -- PTTS_EINVAL when it
 * does not apply (f32, M < 128, the f32 epilogue, or a matrix without a row-major copy such as the lm heads).
 * row_stats: float[2*M] scratch for path 1 with use_ln (may be NULL otherwise).  residual may equal y (in place). */
int ptts_op_linear2(const ptts_decoder_config* cfg, const void* blob, int32_t tensor_id, int32_t index,
                    const void* x, int32_t M, int32_t use_ln, int32_t epilogue /*0 store,1 act,2 +res,3 f32*/,
                    const void* residual, void* y, int32_t path, float* row_stats, void* stream);
/* ptts_op_linear2 with path 0 (the decode GEMM): the original signature, kept for existing callers. */
int ptts_op_linear(const ptts_decoder_config* cfg, const void* blob, int32_t tensor_id, int32_t index,
                   const void* x, int32_t M, int32_t use_ln, int32_t epilogue, const void* residual, void* y, void* stream);
/* The scoring heads of ptts_score over a given residual stream, with no decoder forward in front: the same launch sequence
 * (ptts_score calls the same function).  Test hook for the scoring kernels.
 *   x         [B][P+T][H] in the model dtype: the decoder output; rows P .. P+T-1 of each utterance are the label positions
 *   labels, dec_ids, token_nll, out_logits, codebook_sums   as for ptts_score ([B,T,K], [B*K,T], [B,T,K], [B*K,T,V], [K][2])
 *   path 0    the unfused route: the lm heads GEMM (launch_linear, f32 logits) over the B rows of each frame into
 *             logits_scratch [B*K][V] f32, then score_rows_kernel; every dtype; labels may be NULL (logits only)
 *   path 1    the fused heads + cross-entropy kernel, under ptts_score's rule: bf16, labels given, no out_logits, hidden_size
 *             % 64 == 0 and vocab_size <= 8192, heads_rm from ptts_lm_heads_rowmajor_pack.  xs_scratch [B*T][H] bf16 receives
 *             the gathered label rows and row_stats [B*T][2] f32 their LayerNorm (mean, rstd).
 * PTTS_EINVAL, with nothing launched, when an argument breaks these rules or a scratch buffer the path needs is NULL. */
int ptts_op_score(const ptts_decoder_config* cfg, const void* blob, const void* heads_rm, const void* x, int32_t B, int32_t P,
                  int32_t T, const int64_t* labels, const int64_t* dec_ids, int32_t path, float* token_nll, float* out_logits,
                  float* codebook_sums, void* xs_scratch, float* row_stats, float* logits_scratch, void* stream);
/* Self- or cross-attention of q_len new positions per batch row (ParlerTTSSdpaAttention after the projections, :858-914), with
 * the kernels the decoder launches.  Test hook for the attention sweeps.
 *   dtype PTTS_BF16 / PTTS_F32; nh query heads, nkv K/V heads (nh % nkv == 0); head_dim 64; scale 1/8.
 *   self  (cross == 0): qkv [B*q_len, (nh + 2 nkv)*64] = q | k | v of the new positions, at cache positions past_len .. past_len +
 *                       q_len - 1; the new K (rotary applied) and V rows are appended to the caches; causal over the cache.
 *   cross (cross != 0): qkv = q [B*q_len, nh*64]; keys are the kv_len cached rows; past_len only sets the rotary position.
 *   kcache, vcache [B][nkv][capacity][64], rows stored swizzled (element d of row t at (((d/8) ^ t) % 8)*8 + d%8).
 *   rope != 0: rope_cos / rope_sin [max_pos][64] in dtype, applied to q (and to the appended K rows).
 *   key_mask [B][mask_len] int32 or NULL: key t < mask_len with key_mask[b][t] == 0 is excluded.
 *   prefill_sweep (q_len > 1): 0 = the decoder's choice (the tensor-core sweep for bf16 with nh == nkv),
 *                  1 = always the scalar sweep (attention_item).
 *   out [B*q_len, nh*64] in dtype. */
int ptts_op_attention(int32_t dtype, int32_t B, int32_t nh, int32_t nkv, int32_t q_len, int32_t past_len, int32_t cross,
                      int32_t kv_len, int32_t capacity, int32_t rope, const void* rope_cos, const void* rope_sin, const void* qkv,
                      void* kcache, void* vcache, const int32_t* key_mask, int32_t mask_len, int32_t prefill_sweep, void* out,
                      void* stream);

/* Attention weights of one layer by the eager definition of ptts_generate_set_probes, with the kernel the decoder launches for
 * it.  Test hook.  q: [B*q_len, ldq] with head h at columns h*64 (before RoPE and scaling); kcache [B][nkv][capacity][64]
 * swizzled as for ptts_op_attention; self (cross == 0): query row j sits at position past_len + j and sees keys 0 .. past_len + j
 * of kv_len = past_len + q_len; cross: all kv_len keys.  key_mask as for ptts_op_attention.  out [B][nh][q_len][kv_len]. */
int ptts_op_attention_probs(int32_t dtype, int32_t B, int32_t nh, int32_t nkv, int32_t q_len, int32_t past_len, int32_t cross,
                            int32_t kv_len, int32_t capacity, int32_t rope, const void* rope_cos, const void* rope_sin, const void* q,
                            int64_t ldq, const void* kcache, const int32_t* key_mask, int32_t mask_len, void* out, void* stream);

/* ---- DAC decode ------------------------------------------------------------------------------ */
typedef struct ptts_dac_config {
  int32_t n_codebooks, codebook_size, codebook_dim;
  int32_t latent_dim;          /* DACConfig.latent_dim = 1024 (configuration_dac.py:14) */
  int32_t decoder_dim;         /* 1536 */
  int32_t n_blocks;            /* 4 */
  int32_t strides[8];          /* 8,8,4,2 */
  int32_t dtype;               /* storage dtype of activations/weights: PTTS_BF16 or PTTS_F32 */
  /* encoder (descript-audio-codec Encoder / transformers DacEncoder, modeling_dac.py:442-472); encoder_dim = 0: decode only */
  int32_t encoder_dim;         /* 64: channels after the input conv, doubled by every block */
  int32_t n_enc_blocks;        /* 4 */
  int32_t encoder_rates[8];    /* 2,4,8,8: even, <= 32, product = the decoder hop */
} ptts_dac_config;

int ptts_dac_blob_bytes(const ptts_dac_config* cfg, int64_t* out_bytes);
int ptts_dac_num_tensors(const ptts_dac_config* cfg, int32_t* out);
/* Pack one weight-norm-folded tensor.  `name_id` enumerates tensors in network order; see
 * parler_tts_b200/dac_wrapper.py::_dac_tensor_list for the (id -> state-dict key) table. */
int ptts_dac_pack(const ptts_dac_config* cfg, void* blob, int32_t name_id, const void* src,
                  int32_t src_dtype, int64_t numel, void* stream);
int ptts_dac_workspace_bytes(const ptts_dac_config* cfg, int32_t B, int32_t T, int64_t* out_bytes);
/* DACModel.decode (dac_wrapper/modeling_dac.py:106-142): codes [B, K, T] int64 ->
 * audio [B, 1, hop*T] in cfg->dtype.  = quantizer.from_codes (:138) + model.decode (:139). */
int ptts_dac_decode(const ptts_dac_config* cfg, const void* blob, void* workspace, int64_t workspace_bytes,
                    const int64_t* codes, int32_t B, int32_t T, void* audio_out, void* stream);
/* Same, over a ragged batch: row b holds frame_lengths[b] frames (device int32 [B]; NULL = every row has T, which is
 * ptts_dac_decode).  Row b of audio_out equals the decode of codes[b, :, :n_b] alone, bit for bit, in samples
 * [0, hop*n_b) and is 0 in [hop*n_b, hop*T); codes at frames >= n_b are never read and may hold any value.  The
 * kernels clamp each length to [0, T]; the caller validates them.  The workspace is ptts_dac_workspace_bytes(B, T). */
int ptts_dac_decode2(const ptts_dac_config* cfg, const void* blob, void* workspace, int64_t workspace_bytes,
                     const int64_t* codes, int32_t B, int32_t T, const int32_t* frame_lengths, void* audio_out,
                     void* stream);
/* Windowed decode, for streaming: row b's window is codes[b, :, s_b : s_b + n_b] of codes [B, K, T_codes] (s_b =
 * frame_start[b], n_b = frame_lengths[b]; device int32 [B] each; n_b <= T <= T_codes, s_b + n_b <= T_codes).  It is decoded
 * as ptts_dac_decode2 decodes that window copied alone to frame 0, and audio_out [B, 1, hop*T] holds, bit for bit, that decode's
 * samples [hop*lo_b, hop*hi_b) (lo_b = emit_lo[b], hi_b = emit_hi[b], device int32 [B], 0 <= lo_b <= hi_b <= n_b) and 0
 * everywhere else.  Each layer computes only the rows those samples depend on, so the cost follows the emit ranges, not the
 * windows.  The kernels clamp the values; the caller guarantees that the ids inside the windows are in range.  The workspace
 * is ptts_dac_workspace_bytes(B, T). */
int ptts_dac_decode3(const ptts_dac_config* cfg, const void* blob, void* workspace, int64_t workspace_bytes,
                     const int64_t* codes, int32_t B, int32_t T_codes, int32_t T,
                     const int32_t* frame_start, const int32_t* frame_lengths,
                     const int32_t* emit_lo, const int32_t* emit_hi, void* audio_out, void* stream);

/* ---- DAC encode ------------------------------------------------------------------------------ */
/* The encoder weights (encoder convs and snake alphas, quantizer in_proj, unit-normalised codebooks) live in a second blob
 * with its own tensor table; the decode blob above is unchanged.  All of these fail with PTTS_EINVAL when
 * cfg->encoder_dim == 0, a stride is odd or > 32, or the encoder hop differs from the decoder hop. */
int ptts_dac_encoder_blob_bytes(const ptts_dac_config* cfg, int64_t* out_bytes);
int ptts_dac_encoder_num_tensors(const ptts_dac_config* cfg, int32_t* out);
/* Pack one weight-norm-folded tensor; parler_tts_b200/dac_wrapper.py::_dac_encoder_tensor_list gives the (id -> key)
 * table.  Load-time only (the reference builds these modules in descript's DAC(), dac_wrapper/modeling_dac.py:24-31). */
int ptts_dac_encoder_pack(const ptts_dac_config* cfg, void* enc_blob, int32_t name_id, const void* src,
                          int32_t src_dtype, int64_t numel, void* stream);
int ptts_dac_encode_workspace_bytes(const ptts_dac_config* cfg, int32_t B, int32_t samples, int64_t* out_bytes);
/* DACModel.encode (dac_wrapper/modeling_dac.py:33-104): model.preprocess's right zero-pad to the hop (:64) + model.encode
 * (:95) = encoder + residual vector quantizer over the first n_q codebooks.
 *   audio [B][samples] in cfg->dtype (channel 0 of input_values);  codes_out [B][n_q][ceil(samples / hop)] int64;
 *   latents_out: NULL, or the encoder output [B][T][latent_dim] in cfg->dtype (a test hook).
 * Needs the decode blob too: the quantizer's raw codebooks and out_proj live there. */
int ptts_dac_encode(const ptts_dac_config* cfg, const void* dec_blob, const void* enc_blob, void* workspace,
                    int64_t workspace_bytes, const void* audio, int32_t B, int32_t samples, int32_t n_q, int64_t* codes_out,
                    void* latents_out, void* stream);
/* Same, over a ragged batch: row b holds sample_lengths[b] = n_b samples (device int32 [B]; NULL = every row has `samples`,
 * which is ptts_dac_encode).  Row b of codes_out and latents_out equals the encode of audio[b, :n_b] alone, bit for bit, in
 * frames [0, ceil(n_b / hop)); later frames hold codebook_size in every codebook and zero latents.  Samples at or past n_b are
 * never read and may hold any value.  The kernels clamp each length to [1, samples]; the caller validates them.  The
 * workspace is ptts_dac_encode_workspace_bytes(B, samples). */
int ptts_dac_encode2(const ptts_dac_config* cfg, const void* dec_blob, const void* enc_blob, void* workspace,
                     int64_t workspace_bytes, const void* audio, int32_t B, int32_t samples, const int32_t* sample_lengths,
                     int32_t n_q, int64_t* codes_out, void* latents_out, void* stream);

/* One codec convolution as the decode and encode walks launch it (test hook for the DAC conv kernels).  Activations are
 * channels-last [B][rows][C] in dtype; every buffer belongs to the caller.
 *   kernel 0: conv_kernel (bf16 or f32): out_raw = conv(snake_alpha(x)) + bias (+ res) (tanh when tanh_out); alpha [Cin] or
 *             NULL (no input snake).  samples > 0 (conv_same only): the input has `samples` rows, zeros past them (the
 *             generic encode walk's input conv).
 *   kernel 1: conv_tc_kernel (bf16; PTTS_EINVAL where conv_tc_supported refuses): out_raw = conv(x) + bias (+ res) and/or
 *             out_act = snake_{alpha_next}(that), alpha_next [Cout].  res may equal out_raw (in place).
 *   kernel 2: final_conv_tanh_kernel (bf16, kind 0, Cout 1, taps 7, dil 1, final_conv_supported(Cin)): out_raw = tanh(conv + bias).
 *   kernel 3: enc_input_conv_kernel (bf16, kind 0, Cin 1, taps 7, dil 1): T rows from `samples` <= T waveform samples x [B][samples];
 *             out_raw and out_act = snake_{alpha_next}(out_raw), both required.
 * kind (dil_or_stride = dilation for kind 0, the even stride s otherwise):
 *   0 conv_same(Cin, Cout, T, taps, dil):  Conv1d(k = taps, dilation, "same"), weight [Cout][Cin][taps], T rows in and out;
 *   1 conv_up(Cin, Cout, T, s):            ConvTranspose1d(k = 2s, stride s, pad ceil(s/2)), weight [Cin][Cout][2s], T -> T*s rows;
 *   2 conv_super_rows(Cin, Cout, T, s):    Conv1d(k = 2s, stride s, pad s/2), weight [Cout][Cin][2s], T -> T/s rows (T % s == 0).
 * frame_lengths (device int32 [B], or NULL) and frames: a ragged batch as in ptts_dac_decode2, input and output rows being whole
 * frames (kernels 0-2).  The weight is packed into `scratch` by the blob's pack for that tensor; scratch holds at least
 * (2 * Cin * Cout * k + k * Cin) * dtype size + 256 bytes (k = taps, or 2s).  PTTS_EINVAL for what the kernel or its launcher
 * refuses: taps > 7 or a receptive field wider than conv_kernel's tile, a ragged reach past conv_tc_kernel's zero band, a
 * kernel / dtype / argument combination it does not take. */
int ptts_op_dac_conv(int32_t dtype, int32_t kernel, int32_t kind, int32_t B, int32_t Cin, int32_t Cout, int32_t T, int32_t taps,
                     int32_t dil_or_stride, int32_t samples, const void* weight, const void* bias, const void* alpha,
                     const void* alpha_next, const void* x, const void* res, void* out_raw, void* out_act, int32_t tanh_out,
                     const int32_t* frame_lengths, int32_t frames, void* scratch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PTTS_B200_H */
