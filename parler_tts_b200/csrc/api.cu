// api.cu -- the C ABI (include/ptts_b200.h): argument validation, weight packing, the generation
// session (prefill / decode step / sample / CUDA-graph replay); the DAC entry points call the codec walks of dac.cu / dac_enc.cu.
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "common.cuh"
#include "dac.h"
#include "kernels.h"
#include "layout.h"
#include "step.h"

namespace ptts {
static thread_local std::string g_err;
void set_error(const std::string& m) { g_err = m; }
int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
static bool env_flag(const char* name, bool dflt) {
  const char* v = getenv(name);
  if (!v || !*v) return dflt;
  return !(v[0] == '0' || v[0] == 'n' || v[0] == 'N' || v[0] == 'f' || v[0] == 'F');
}
}  // namespace ptts

using namespace ptts;

// How a session runs its decode steps; ptts_session_fused reports the value.
enum DecodePath {
  DECODE_MULTI_KERNEL = 0,  // 8L+3 kernels per token, replayed from a CUDA graph
  DECODE_STEP = 1,          // one persistent kernel per token (step.cu)
  DECODE_CLUSTER = 2,       // the cluster variant of that kernel (step2.cu: 6 device-wide phases per layer)
};

// ptts_generate_set_probes: slot s of each output at ptr + s * *_step elements (model dtype)
struct ProbeWindow {
  void* self_attn; void* cross_attn; void* hidden;
  int first_step, n_steps;
  int64_t self_ld, self_step, cross_step, hidden_step;
};

// ptts_generate_set_alignment: rows [first_row, first_row + n_rows) of out [n_rows][B][key_len] fp32
struct AlignWindow {
  const int32_t* heads; int n_heads;   // device [n_heads][2] (layer, head)
  std::vector<int> layer_heads;        // entries per layer (host copy of the list's layers)
  int key0, key_len;
  float* out;
  int first_row, n_rows;
};

struct ptts_session {
  ptts_decoder_config cfg;
  DecoderLayout L;
  WorkspaceLayout W;
  const char* blob;
  char* ws;
  int sm_count;
  bool has_prompt_mask, has_enc_mask, begun, prefilled;
  ptts_gen_params gen;
  int n0;            // decoder input columns of the current generate() call (1: the BOS column; > 1: continuing from codes)
  bool ragged;       // the call's rows continue from inputs of different lengths (ptts_generate_begin_ids2): W.row_shift is live
  int sampled;       // ptts_sample / ptts_op_sample_phase calls since the last ptts_prefill
  bool decoded;      // a decode step ran since the last ptts_prefill (the cache holds positions past P + n0)
  bool slots;        // slot mode (ptts_generate_set_slots): ragged, and every row is a request with its own column and Philox key
  cudaStream_t cap_stream;
  cudaGraphExec_t exec;
  bool graph_ready;
  int64_t launches;  // kernels launched through this session (bench.py reports it)
  long long* prof;
  DecodePath path;
  StepParams sp;     // the step kernels' parameters (DECODE_STEP, DECODE_CLUSTER)
  ptts_sampling_ext ext;  // ptts_generate_set_sampling_ext; off after every ptts_generate_begin*
  ptts_logits_ext lext;   // ptts_generate_set_logits_ext; off after every ptts_generate_begin*
  SampleOut out;          // ptts_generate_set_outputs; off (both pointers null) after every ptts_generate_begin*
  ProbeWindow probe;      // ptts_generate_set_probes; off (all pointers null) after every ptts_generate_begin*
  AlignWindow align;      // ptts_generate_set_alignment; off (out null) after every ptts_generate_begin*
  int64_t graph_launches; // kernels of one replay of the captured decode graph
};

static const ptts_sampling_ext kExtOff = {0, 0.f, 1.f, 0.f, 0.f};
// the sampler with the ptts_sampling_ext stages, or nullptr while none of them changes the result
static const ptts_sampling_ext* active_ext(const ptts_session* s) {
  const ptts_sampling_ext& x = s->ext;
  const bool warp = s->gen.do_sample && (x.min_p > 0.f || x.typical_p < 1.f || x.epsilon_cutoff > 0.f || x.eta_cutoff > 0.f);
  return (x.no_repeat_ngram_size > 0 || warp) ? &s->ext : nullptr;
}
// the ptts_logits_ext stages, or nullptr while none is set
static const ptts_logits_ext* active_lext(const ptts_session* s) {
  const ptts_logits_ext& x = s->lext;
  const bool on = x.bias1 != nullptr || x.n_seq > 0 || x.forced_bos_token_id >= 0 || x.forced_eos_token_id >= 0 ||
                  x.remove_invalid_values || x.decay != nullptr || x.suppress != nullptr || x.begin_suppress != nullptr ||
                  x.renormalize_logits;
  return on ? &s->lext : nullptr;
}
// the per-step outputs, or nullptr while none is set
static const SampleOut* active_out(const ptts_session* s) {
  return (s->out.logits != nullptr || s->out.scores != nullptr) ? &s->out : nullptr;
}
// the attention / hidden-state window, or nullptr while none is set
static const ProbeWindow* active_probe(const ptts_session* s) {
  const ProbeWindow& w = s->probe;
  return (w.self_attn != nullptr || w.cross_attn != nullptr || w.hidden != nullptr) ? &w : nullptr;
}
// the alignment window, or nullptr while none is set
static const AlignWindow* active_align(const ptts_session* s) { return s->align.out != nullptr ? &s->align : nullptr; }
// the path decode steps take now: a probe or alignment window needs the per-layer kernels of the multi-kernel path
static DecodePath decode_path(const ptts_session* s) {
  return (active_probe(s) != nullptr || active_align(s) != nullptr) ? DECODE_MULTI_KERNEL : s->path;
}

// the knobs of the EXT sampler, or nullptr for the plain one: the outputs, the ptts_logits_ext stages and slot mode run on the EXT
// sampler, with every ptts_sampling_ext stage off when none is active (it then computes what the plain sampler computes)
static const ptts_sampling_ext* sampler_ext(const ptts_session* s) {
  const ptts_sampling_ext* x = active_ext(s);
  return (x == nullptr && (active_out(s) != nullptr || active_lext(s) != nullptr || s->slots)) ? &kExtOff : x;
}
// slot mode's per-row Philox keys, or nullptr
static const int* slot_keys(const ptts_session* s) { return s->slots ? (const int*)(s->ws + s->W.row_key) : nullptr; }
static const int* slot_max_lens(const ptts_session* s) { return s->slots ? (const int*)(s->ws + s->W.row_max_len) : nullptr; }

extern "C" {

const char* ptts_last_error(void) { return g_err.c_str(); }
int ptts_version(void) { return 100; }

// ---- weights ------------------------------------------------------------------------------------
int ptts_decoder_blob_bytes(const ptts_decoder_config* cfg, int64_t* out_bytes) {
  PTTS_REQUIRE(cfg && out_bytes, "null argument");
  if (int e = validate_config(*cfg)) return e;
  *out_bytes = make_layout(*cfg).total;
  return PTTS_OK;
}

int ptts_decoder_pack(const ptts_decoder_config* cfg, void* blob, int32_t tensor_id, int32_t index, const void* src,
                      int32_t src_dtype, int64_t rows, int64_t cols, void* stream) {
  PTTS_REQUIRE(cfg && blob && src, "null argument");
  if (int e = validate_config(*cfg)) return e;
  PTTS_REQUIRE(src_dtype == PTTS_BF16 || src_dtype == PTTS_F32, "pack: src dtype must be bf16 or f32");
  const DecoderLayout L = make_layout(*cfg);
  cudaStream_t st = (cudaStream_t)stream;
  char* base = (char*)blob;
  MatSlot ms;
  const bool per_layer = (tensor_id >= PTTS_T_LN1_W && tensor_id <= PTTS_T_FC2);
  if (per_layer) PTTS_REQUIRE(index >= 0 && index < L.L, "pack: layer %d out of range", index);
  if (matrix_slot(L, tensor_id, index, &ms)) {
    if (tensor_id == PTTS_T_LM_HEAD) PTTS_REQUIRE(index >= 0 && index < L.K, "pack: codebook %d out of range", index);
    PTTS_REQUIRE(cols == ms.m.K, "pack: tensor %d expects %d columns, got %lld", tensor_id, ms.m.K, (long long)cols);
    PTTS_REQUIRE(rows > 0 && ms.row_off + rows <= ms.m.N, "pack: tensor %d rows %lld do not fit fused matrix of %d rows", tensor_id, (long long)rows, ms.m.N);
    return pack_matrix(src, src_dtype, rows, cols, ms.row_off, ms.m.K, base + ms.m.w, cfg->dtype, st);
  }
  const int H = L.H;
  switch (tensor_id) {
    case PTTS_T_EMBED_TOKENS:
      PTTS_REQUIRE(index >= 0 && index < L.K && rows == L.V + 1 && cols == H, "pack: embed_tokens shape");
      return pack_plain(src, src_dtype, rows * cols, base + L.embed + (int64_t)index * (L.V + 1) * H * L.es, cfg->dtype, st);
    case PTTS_T_POS_TABLE:
      PTTS_REQUIRE(!cfg->rope && rows == cfg->max_positions && cols == H, "pack: pos table shape");
      return pack_plain(src, src_dtype, rows * cols, base + L.pos, cfg->dtype, st);
    case PTTS_T_ROPE_COS:
    case PTTS_T_ROPE_SIN:
      PTTS_REQUIRE(cfg->rope && rows == cfg->max_positions && cols == PTTS_HEAD_DIM, "pack: rope table shape");
      return pack_plain(src, src_dtype, rows * cols, base + (tensor_id == PTTS_T_ROPE_COS ? L.rope_cos : L.rope_sin), cfg->dtype, st);
    case PTTS_T_LN1_W: case PTTS_T_LN1_B: case PTTS_T_LN2_W: case PTTS_T_LN2_B: case PTTS_T_LN3_W: case PTTS_T_LN3_B:
    case PTTS_T_FINAL_LN_W: case PTTS_T_FINAL_LN_B: {   // the LayerNorm in front of a matrix
      PTTS_REQUIRE(rows * cols == H, "pack: LayerNorm parameter must have %d elements", H);
      const int m = tensor_id <= PTTS_T_LN1_B ? MAT_QKV : tensor_id <= PTTS_T_LN2_B ? MAT_Q_CROSS : tensor_id <= PTTS_T_LN3_B ? MAT_FC1 : MAT_HEADS;
      const DecoderMatrix dm = decoder_matrix(L, m, index);
      const bool gamma = tensor_id == PTTS_T_LN1_W || tensor_id == PTTS_T_LN2_W || tensor_id == PTTS_T_LN3_W || tensor_id == PTTS_T_FINAL_LN_W;
      return pack_plain(src, src_dtype, H, base + (gamma ? dm.ln_w : dm.ln_b), PTTS_F32, st);
    }
    default:
      return fail(PTTS_EINVAL, "pack: unknown tensor id %d", tensor_id);
  }
}

int ptts_decoder_finalize(const ptts_decoder_config* cfg, void* blob, void* stream) {
  PTTS_REQUIRE(cfg && blob, "null argument");
  if (int e = validate_config(*cfg)) return e;
  if (cfg->dtype != PTTS_BF16) return PTTS_OK;  // the f32 path applies LayerNorm explicitly
  const DecoderLayout L = make_layout(*cfg);
  cudaStream_t st = (cudaStream_t)stream;
  char* b = (char*)blob;
  for (int m = 0; m < MAT_COUNT; m++)
    for (int i = 0; i < (m == MAT_HEADS ? 1 : L.L); i++) {
      const DecoderMatrix d = decoder_matrix(L, m, i);
      if (d.ln_w >= 0) {
        float* c = (float*)(b + d.c);
        if (int e = fold_layernorm(b + d.w, d.N, d.K, (const float*)(b + d.ln_w), (const float*)(b + d.ln_b), c, c + d.N, st)) return e;
      }
      // the row-major copy for the wgmma prefill GEMM (gemm_tc.cu) is unpacked after the fold
      if (d.rm >= 0)
        if (int e = unpack_fragments(b + d.w, b + d.rm, d.N, d.K, st)) return e;
    }
  if (L.cl_NC > 0) {  // second copy of the layer matrices, sliced per (phase, cluster, rank) for the cluster step kernel (step2.cu)
    for (int i = 0; i < L.L; i++)
      if (int e = cluster_pack_layer(L, b + L.layer0 + L.layer_stride * i, st)) return e;
  }
  return PTTS_OK;
}

int ptts_workspace_bytes3(const ptts_decoder_config* cfg, int32_t B, int32_t P, int32_t S, int32_t max_cache_len, int32_t max_input_len,
                          int32_t takes, int64_t* out_bytes) {
  PTTS_REQUIRE(cfg && out_bytes, "null argument");
  if (int e = validate_config(*cfg)) return e;
  PTTS_REQUIRE(B > 0 && P >= 0 && S > 0 && max_cache_len > P, "workspace: need B>0, P>=0, S>0, max_cache_len>P (got %d %d %d %d)", B, P, S, max_cache_len);
  PTTS_REQUIRE(max_input_len >= 1 && max_input_len < max_cache_len - P + 1, "workspace: max_input_len %d must be in [1, max_cache_len - P]", max_input_len);
  PTTS_REQUIRE(takes >= 1 && B % takes == 0, "workspace: takes %d must be >= 1 and divide B = %d", takes, B);
  *out_bytes = make_workspace(*cfg, B, P, S, max_cache_len, max_input_len, takes).total;
  return PTTS_OK;
}

int ptts_workspace_bytes2(const ptts_decoder_config* cfg, int32_t B, int32_t P, int32_t S, int32_t max_cache_len, int32_t max_input_len,
                          int64_t* out_bytes) {
  return ptts_workspace_bytes3(cfg, B, P, S, max_cache_len, max_input_len, 1, out_bytes);
}

int ptts_workspace_bytes(const ptts_decoder_config* cfg, int32_t B, int32_t P, int32_t S, int32_t max_cache_len, int64_t* out_bytes) {
  return ptts_workspace_bytes2(cfg, B, P, S, max_cache_len, 1, out_bytes);
}

// ---- session ------------------------------------------------------------------------------------
int ptts_session_create3(const ptts_decoder_config* cfg, const void* blob, void* workspace, int64_t workspace_bytes,
                         int32_t B, int32_t P, int32_t S, int32_t max_cache_len, int32_t max_input_len, int32_t takes, ptts_session** out) {
  PTTS_REQUIRE(cfg && blob && workspace && out, "null argument");
  if (int e = validate_config(*cfg)) return e;
  PTTS_REQUIRE(B > 0 && P >= 0 && S > 0 && max_cache_len > P, "session: bad shape B=%d P=%d S=%d Tmax=%d", B, P, S, max_cache_len);
  PTTS_REQUIRE(max_cache_len <= cfg->max_positions, "session: cache length %d exceeds max_position_embeddings %d", max_cache_len, cfg->max_positions);
  PTTS_REQUIRE(max_input_len >= 1 && max_input_len < max_cache_len - P + 1, "session: max_input_len %d must be in [1, max_cache_len - P]", max_input_len);
  PTTS_REQUIRE(takes >= 1 && B % takes == 0, "session: takes %d must be >= 1 and divide B = %d", takes, B);
  ptts_session* s = new (std::nothrow) ptts_session();
  PTTS_REQUIRE(s, "out of host memory");
  s->cfg = *cfg;
  s->L = make_layout(*cfg);
  s->W = make_workspace(*cfg, B, P, S, max_cache_len, max_input_len, takes);
  s->n0 = 1;
  s->ragged = s->slots = false;
  s->ext = kExtOff;
  s->lext = kLogitsExtOff;
  s->out = SampleOut{};
  s->probe = ProbeWindow{};
  s->graph_launches = 0;
  if (workspace_bytes < s->W.total) {
    int64_t need = s->W.total;
    delete s;
    return fail(PTTS_EINVAL, "session: workspace too small (%lld < %lld bytes)", (long long)workspace_bytes, (long long)need);
  }
  s->blob = (const char*)blob;
  s->ws = (char*)workspace;
  int dev = 0;
  cudaGetDevice(&dev);
  s->sm_count = 132;
  cudaDeviceGetAttribute(&s->sm_count, cudaDevAttrMultiProcessorCount, dev);
  s->graph_ready = false;
  s->exec = nullptr;
  s->cap_stream = nullptr;
  s->begun = s->prefilled = false;
  s->path = DECODE_MULTI_KERNEL;
  s->prof = nullptr;
  s->launches = 0;
  *out = s;
  return PTTS_OK;
}

int ptts_session_create2(const ptts_decoder_config* cfg, const void* blob, void* workspace, int64_t workspace_bytes,
                         int32_t B, int32_t P, int32_t S, int32_t max_cache_len, int32_t max_input_len, ptts_session** out) {
  return ptts_session_create3(cfg, blob, workspace, workspace_bytes, B, P, S, max_cache_len, max_input_len, 1, out);
}

int ptts_session_create(const ptts_decoder_config* cfg, const void* blob, void* workspace, int64_t workspace_bytes,
                        int32_t B, int32_t P, int32_t S, int32_t max_cache_len, ptts_session** out) {
  return ptts_session_create2(cfg, blob, workspace, workspace_bytes, B, P, S, max_cache_len, 1, out);
}

int ptts_session_destroy(ptts_session* s) {
  if (!s) return PTTS_OK;
  if (s->exec) cudaGraphExecDestroy(s->exec);
  if (s->cap_stream) cudaStreamDestroy(s->cap_stream);
  delete s;
  return PTTS_OK;
}

// The captured decode graph holds the session's settings and windows by value: drop it, and the next ptts_decode_steps captures
// again.
static void drop_graph(ptts_session* s) {
  if (s->exec) cudaGraphExecDestroy(s->exec);
  s->exec = nullptr;
  s->graph_ready = false;
}

static SampleArgs sample_args(ptts_session* s) {
  SampleArgs a{};
  const WorkspaceLayout& W = s->W;
  a.logits = (const float*)(s->ws + W.logits);
  a.scores = (float*)(s->ws + W.scores);
  a.raw_ids = (int64_t*)(s->ws + W.raw_ids);
  a.raw_ld = W.raw_ld;
  a.cur_ids = (int*)(s->ws + W.cur_ids);
  a.eos_seen = (int*)(s->ws + W.eos_seen);
  a.unfinished = (int*)(s->ws + W.unfinished);
  a.first_unf = (int*)(s->ws + W.first_unf);
  a.ctrl = (Ctrl*)(s->ws + W.ctrl);
  a.gen = (const ptts_gen_params*)(s->ws + W.gen);
  a.prefix_cells = W.prefix_cells >= 0 ? (int64_t*)(s->ws + W.prefix_cells) : nullptr;
  a.shift = s->ragged ? (int*)(s->ws + W.row_shift) : nullptr;
  a.B = W.B; a.K = s->cfg.num_codebooks; a.V = s->cfg.vocab_size;
  a.bos = s->cfg.bos_token_id; a.pad = s->cfg.pad_token_id; a.eos = s->cfg.eos_token_id;
  return a;
}


// The step kernels cover bf16, B <= 32, K <= 16: anything else runs the 8L+3-kernel path -- a 2x slower step.  Say so once per
// process instead of degrading silently (ptts_session_fused reports which path a session uses).
static DecodePath step_declined(ptts_session* s, const char* why) {
  static bool warned = false;
  if (!warned) {
    fprintf(stderr, "ptts_b200: fused decode step not used for this session (B=%d, H=%d, K=%d: %s); decode steps run the multi-kernel path\n",
            s->W.B, s->L.H, s->L.K, why);
    warned = true;
  }
  return DECODE_MULTI_KERNEL;
}

// The fastest decode path the session's shape and the device allow; fills s->sp for the step kernels.  PTTS_FUSED=0 keeps the
// multi-kernel path and PTTS_STEP=legacy keeps step.cu where step2.cu applies: each is the bit-exact reference of the next.
static DecodePath choose_decode_path(ptts_session* s) {
  const ptts_decoder_config& c = s->cfg;
  const DecoderLayout& L = s->L;
  const WorkspaceLayout& W = s->W;
  if (c.dtype != PTTS_BF16 || !env_flag("PTTS_FUSED", true)) return DECODE_MULTI_KERNEL;
  if (W.B > 32 || L.K > 16 || L.H % 64 != 0 || L.F % L.H != 0) return step_declined(s, "batch > 32 rows, > 16 codebooks or an unsupported width");
  StepParams& p = s->sp;
  memset(&p, 0, sizeof(p));
  p.B = W.B; p.H = L.H; p.F = L.F; p.V = L.V; p.K = L.K; p.L = L.L; p.nh = L.nh; p.nkv = L.nkv; p.nckv = L.nckv;
  p.S = W.S; p.P = W.P; p.Tmax = W.Tmax; p.takes = W.takes; p.rope = c.rope; p.act = c.activation; p.qkv_rows = L.qkv_rows; p.ckv_rows = L.ckv_rows;
  p.eps = c.layer_norm_eps; p.scale = 0.125f;
  p.blob = s->blob;
  p.lay = L;
  char* ws = s->ws;
  p.x = (bf16*)(ws + W.img_x); p.qkv = (bf16*)(ws + W.qkv); p.attn = (bf16*)(ws + W.img_attn); p.qc = (bf16*)(ws + W.qc); p.hbuf = (bf16*)(ws + W.img_h);
  p.logits = (float*)(ws + W.logits);
  p.cross_kv = ws + W.cross_kv; p.cross_layer_stride = W.cross_layer_stride;
  p.self_kv = ws + W.self_kv; p.self_layer_stride = W.self_layer_stride;
  p.prompt_mask = s->has_prompt_mask ? (const int*)(ws + W.prompt_mask) : nullptr;
  p.enc_mask = s->has_enc_mask ? (const int*)(ws + W.enc_mask) : nullptr;
  p.sa = sample_args(s);
  p.bar = ((Ctrl*)(ws + W.ctrl))->bar;
  p.progress = (int*)(ws + W.progress);
  if (const char* why = plan_decode_step(p, s->sm_count)) return step_declined(s, why);
  p.do_sample_phase = 1;
  p.prof = s->prof;
  p.cl_x = (bf16*)(ws + W.cl_x); p.cl_attn = (bf16*)(ws + W.cl_attn); p.cl_h = (bf16*)(ws + W.cl_h);
  const char* mode = getenv("PTTS_STEP");
  if (L.cl_NC > 0 && !(mode && strcmp(mode, "legacy") == 0) && cluster_step_available(p)) return DECODE_CLUSTER;
  return DECODE_STEP;
}

int ptts_generate_begin_ids2(ptts_session* s, const ptts_gen_params* gen, const int64_t* input_ids, int32_t n0, const int32_t* input_lens,
                             void* stream) {
  PTTS_REQUIRE(s && gen, "null argument");
  PTTS_REQUIRE(n0 >= 1 && n0 <= s->W.max_input, "generate: %d decoder input columns, the session takes 1 .. %d", n0, s->W.max_input);
  PTTS_REQUIRE(input_ids != nullptr || n0 == 1, "generate: input_ids is required for %d input columns", n0);
  PTTS_REQUIRE(gen->max_length >= 2, "generate: max_length must be >= 2, got %d", gen->max_length);
  PTTS_REQUIRE(gen->max_length <= s->W.raw_ld, "generate: max_length %d exceeds the session's capacity %lld", gen->max_length, (long long)s->W.raw_ld);
  PTTS_REQUIRE(!gen->do_sample || gen->temperature > 0.f, "`temperature` has to be a strictly positive float, got %f", gen->temperature);
  PTTS_REQUIRE(gen->top_k >= 0, "`top_k` has to be a non-negative integer");
  PTTS_REQUIRE(s->cfg.eos_token_id >= 0 && s->cfg.eos_token_id < s->cfg.vocab_size, "eos_token_id out of vocabulary");
  PTTS_REQUIRE(n0 < gen->max_length, "generate: %d input columns leave nothing to generate within max_length %d", n0, gen->max_length);
  cudaStream_t st = (cudaStream_t)stream;
  if (input_lens != nullptr) {   // checked here, once per call: every kernel after the begin trusts the shifts it derives
    PTTS_REQUIRE(input_ids != nullptr, "generate: input_lens needs input_ids");
    std::vector<int32_t> lens(s->W.B);
    PTTS_CHECK_CUDA(cudaMemcpyAsync(lens.data(), input_lens, lens.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PTTS_CHECK_CUDA(cudaStreamSynchronize(st));
    for (int b = 0; b < s->W.B; b++)
      PTTS_REQUIRE(lens[b] >= 1 && lens[b] <= n0, "generate: input_lens[%d] = %d is outside [1, n0 = %d]", b, lens[b], n0);
  }
  // n0 == 1: every length is 1 and every offset 0 -- a uniform batch (and a session without max_input_len > 1 has no row_shift)
  s->ragged = input_lens != nullptr && n0 > 1;
  s->slots = false;
  s->gen = *gen;
  s->gen.input_len = n0;
  s->n0 = n0;
  s->ext = kExtOff;
  s->lext = kLogitsExtOff;
  s->out = SampleOut{};
  if (active_probe(s) || active_align(s)) drop_graph(s);
  s->probe = ProbeWindow{};
  s->align = AlignWindow{};
  PTTS_CHECK_CUDA(cudaMemcpyAsync(s->ws + s->W.gen, &s->gen, sizeof(ptts_gen_params), cudaMemcpyHostToDevice, st));
  if (int e = launch_generate_begin(sample_args(s), input_ids, n0, gen->max_length, s->ragged ? input_lens : nullptr, st)) return e;
  s->begun = true;
  s->prefilled = false;
  return PTTS_OK;
}

int ptts_generate_begin_ids(ptts_session* s, const ptts_gen_params* gen, const int64_t* input_ids, int32_t n0, void* stream) {
  return ptts_generate_begin_ids2(s, gen, input_ids, n0, nullptr, stream);
}

int ptts_generate_begin(ptts_session* s, const ptts_gen_params* gen, void* stream) {
  return ptts_generate_begin_ids(s, gen, nullptr, 1, stream);
}

int ptts_generate_set_sampling_ext(ptts_session* s, const ptts_sampling_ext* ext) {
  PTTS_REQUIRE(s, "null argument");
  if (!s->begun) return fail(PTTS_ESTATE, "ptts_generate_set_sampling_ext called before ptts_generate_begin");
  const ptts_sampling_ext x = ext ? *ext : kExtOff;
  PTTS_REQUIRE(x.no_repeat_ngram_size >= 0, "`no_repeat_ngram_size` has to be a non-negative integer, got %d", x.no_repeat_ngram_size);
  PTTS_REQUIRE(x.min_p >= 0.f && x.min_p <= 1.f, "`min_p` has to be a float in the [0, 1] interval, got %f", x.min_p);
  PTTS_REQUIRE(x.typical_p > 0.f && x.typical_p <= 1.f, "`typical_p` has to be a float in (0, 1] (1 = off), got %f", x.typical_p);
  PTTS_REQUIRE(x.epsilon_cutoff >= 0.f && x.epsilon_cutoff < 1.f, "`epsilon_cutoff` has to be a float in [0, 1) (0 = off), got %f", x.epsilon_cutoff);
  PTTS_REQUIRE(x.eta_cutoff >= 0.f && x.eta_cutoff < 1.f, "`eta_cutoff` has to be a float in [0, 1) (0 = off), got %f", x.eta_cutoff);
  s->ext = x;
  // the knobs are a by-value argument of the captured graph's sampler node: capture again
  drop_graph(s);
  return PTTS_OK;
}

int ptts_generate_set_logits_ext(ptts_session* s, const ptts_logits_ext* ext) {
  PTTS_REQUIRE(s, "null argument");
  if (!s->begun) return fail(PTTS_ESTATE, "ptts_generate_set_logits_ext called before ptts_generate_begin");
  const ptts_logits_ext x = ext ? *ext : kLogitsExtOff;
  const int V = s->cfg.vocab_size;
  PTTS_REQUIRE(x.n_seq >= 0 && x.n_seq <= PTTS_SEQ_BIAS_MAX, "`sequence_bias`: %d sequences of two or more ids, at most %d are supported", x.n_seq, PTTS_SEQ_BIAS_MAX);
  PTTS_REQUIRE(x.n_seq == 0 || (x.seq != nullptr && x.seq_bias != nullptr), "`sequence_bias`: n_seq > 0 needs the seq and seq_bias tables");
  PTTS_REQUIRE(x.forced_bos_token_id >= -1 && x.forced_bos_token_id < V, "`forced_bos_token_id` %d is outside the vocabulary [0, %d)", x.forced_bos_token_id, V);
  PTTS_REQUIRE(x.forced_eos_token_id >= -1 && x.forced_eos_token_id < V, "`forced_eos_token_id` %d is outside the vocabulary [0, %d)", x.forced_eos_token_id, V);
  PTTS_REQUIRE(x.decay == nullptr || x.decay_start >= 0, "`exponential_decay_length_penalty`: regulation start %d must be >= 0", x.decay_start);
  PTTS_REQUIRE(x.begin_suppress == nullptr || x.begin_index >= 1, "`begin_suppress_tokens`: begin index %d must be >= 1", x.begin_index);
  s->lext = x;
  // the struct is a by-value argument of the captured graph's sampler node: capture again
  drop_graph(s);
  return PTTS_OK;
}

int ptts_generate_set_outputs(ptts_session* s, float* logits, float* scores, int32_t first_step, int32_t n_steps, int64_t step_stride) {
  PTTS_REQUIRE(s, "null argument");
  if (!s->begun) return fail(PTTS_ESTATE, "ptts_generate_set_outputs called before ptts_generate_begin");
  PTTS_REQUIRE(first_step >= 0 && n_steps >= 0, "outputs: the window needs first_step >= 0 and n_steps >= 0, got %d and %d", first_step, n_steps);
  SampleOut o{};
  if (logits != nullptr || scores != nullptr) {
    const int64_t rows = (int64_t)s->W.B * s->cfg.num_codebooks * s->cfg.vocab_size;
    PTTS_REQUIRE(step_stride >= rows, "outputs: step_stride %lld is below the session's B*K*V = %lld floats", (long long)step_stride, (long long)rows);
    o = SampleOut{logits, scores, first_step, n_steps, step_stride};
  }
  const bool same = o.logits == s->out.logits && o.scores == s->out.scores && o.first_step == s->out.first_step &&
                    o.n_steps == s->out.n_steps && o.step_stride == s->out.step_stride;
  s->out = o;
  // the window is a by-value argument of the captured graph's sampler node: capture again when it moved
  if (!same) drop_graph(s);
  return PTTS_OK;
}

int ptts_generate_set_probes(ptts_session* s, void* self_attn, void* cross_attn, void* hidden, int32_t first_step, int32_t n_steps,
                             int64_t self_ld, int64_t self_step, int64_t cross_step, int64_t hidden_step) {
  PTTS_REQUIRE(s, "null argument");
  PTTS_REQUIRE(first_step >= 0 && n_steps >= 0, "probes: the window needs first_step >= 0 and n_steps >= 0, got %d and %d", first_step, n_steps);
  ProbeWindow w{};
  if (self_attn != nullptr || cross_attn != nullptr || hidden != nullptr) {
    PTTS_REQUIRE(!s->ragged, "probes: the probe kernels take one position for the whole batch, not a ragged continuation's");
    const WorkspaceLayout& W = s->W;
    const DecoderLayout& L = s->L;
    // (the prefill slot's row count P + n0 is only known when ptts_prefill / ptts_score runs: run_forward checks self_ld there)
    PTTS_REQUIRE(first_step > 0 || n_steps <= 1, "probes: the prefill slot (step 0) takes a window of its own (n_steps 1)");
    const int64_t longest = W.P + s->n0 + first_step + (int64_t)n_steps - 1;
    PTTS_REQUIRE(self_attn == nullptr || first_step == 0 || self_ld >= longest, "probes: self_ld %lld is below the window's %lld keys",
                 (long long)self_ld, (long long)longest);
    PTTS_REQUIRE(self_attn == nullptr || n_steps <= 1 || self_step >= (int64_t)L.L * W.B * L.nh * self_ld, "probes: self_step is below one slot");
    PTTS_REQUIRE(cross_attn == nullptr || n_steps <= 1 || cross_step >= (int64_t)L.L * W.B * L.nh * W.S, "probes: cross_step is below one slot");
    PTTS_REQUIRE(hidden == nullptr || n_steps <= 1 || hidden_step >= (int64_t)(L.L + 1) * W.B * L.H, "probes: hidden_step is below one slot");
    w = ProbeWindow{self_attn, cross_attn, hidden, first_step, n_steps, self_ld, self_step, cross_step, hidden_step};
  }
  const ProbeWindow& o = s->probe;
  const bool same = w.self_attn == o.self_attn && w.cross_attn == o.cross_attn && w.hidden == o.hidden && w.first_step == o.first_step &&
                    w.n_steps == o.n_steps && w.self_ld == o.self_ld && w.self_step == o.self_step && w.cross_step == o.cross_step &&
                    w.hidden_step == o.hidden_step;
  s->probe = w;
  // the window is a by-value argument of the captured graph's probe nodes (and it switches the path): capture again when it moved
  if (!same) drop_graph(s);
  return PTTS_OK;
}

int ptts_generate_set_alignment(ptts_session* s, const int32_t* heads, int32_t n_heads, int32_t key0, int32_t key_len, float* out,
                                int32_t first_step, int32_t n_steps) {
  PTTS_REQUIRE(s, "null argument");
  PTTS_REQUIRE(first_step >= 0 && n_steps >= 0, "alignment: the window needs first_step >= 0 and n_steps >= 0, got %d and %d", first_step, n_steps);
  AlignWindow w{};
  if (out != nullptr) {
    PTTS_REQUIRE(!s->ragged, "alignment: the probe kernels take one position for the whole batch, not a ragged continuation's");
    const DecoderLayout& L = s->L;
    // a session with a self-attention prompt prefix aligns to it; one without (prompt_cross_attention) to its cross keys
    const int keys = s->W.P > 0 ? s->W.P : s->W.S;
    PTTS_REQUIRE(heads != nullptr && n_heads > 0, "alignment: the head list is empty");
    PTTS_REQUIRE(key0 >= 0 && key_len > 0 && key0 + key_len <= keys, "alignment: keys [%d, %d) are outside the session's %d %s keys",
                 key0, key0 + key_len, keys, s->W.P > 0 ? "prompt-prefix" : "cross-attention");
    std::vector<int32_t> h(2 * (size_t)n_heads);
    PTTS_CHECK_CUDA(cudaMemcpy(h.data(), heads, h.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    w.layer_heads.assign(L.L, 0);
    std::vector<char> seen((size_t)L.L * L.nh, 0);
    for (int e = 0; e < n_heads; e++) {
      const int l = h[2 * e], hd = h[2 * e + 1];
      PTTS_REQUIRE(l >= 0 && l < L.L && hd >= 0 && hd < L.nh, "alignment: head [%d, %d] is outside %d layers x %d heads", l, hd, L.L, L.nh);
      PTTS_REQUIRE(!seen[(size_t)l * L.nh + hd], "alignment: head [%d, %d] is listed twice", l, hd);
      seen[(size_t)l * L.nh + hd] = 1;
      w.layer_heads[l]++;
    }
    w.heads = heads; w.n_heads = n_heads; w.key0 = key0; w.key_len = key_len; w.out = out;
    w.first_row = first_step; w.n_rows = n_steps;
  }
  const AlignWindow& o = s->align;
  const bool same = w.out == o.out && w.heads == o.heads && w.n_heads == o.n_heads && w.layer_heads == o.layer_heads &&
                    w.key0 == o.key0 && w.key_len == o.key_len && w.first_row == o.first_row && w.n_rows == o.n_rows;
  s->align = w;
  // the window is a by-value argument of the captured graph's alignment nodes (and it switches the path): capture again
  if (!same) drop_graph(s);
  return PTTS_OK;
}

// one decoder pass over q_len new positions per batch row (q_len = P+n0 at prefill, 1 at decode); heads == false stops after
// the last layer and leaves the residual stream x [B][q_len][H] for the caller (ptts_score)
static int run_forward(ptts_session* s, cudaStream_t st, bool prefill, const void* prompt_hidden, const void* enc_hidden,
                       bool heads = true) {
  const ptts_decoder_config& c = s->cfg;
  const DecoderLayout& L = s->L;
  const WorkspaceLayout& W = s->W;
  const int B = W.B, P = W.P, S = W.S, H = L.H, D = PTTS_HEAD_DIM;
  const int n_desc = B / W.takes;   // descriptions: the cross K/V and the encoder mask hold one item each
  const int q_len = prefill ? P + s->n0 : 1;
  const int M = B * q_len;
  const bool pdl = !prefill;  // the one-off prefill stays on plain stream order
  const Ctrl* ctrl = prefill ? nullptr : (const Ctrl*)(s->ws + W.ctrl);
  const int es = L.es;
  char* ws = s->ws;
  const char* blob = s->blob;

  EmbedArgs ea{};
  ea.tables = blob + L.embed;
  ea.pos = c.rope ? nullptr : blob + L.pos;
  ea.prefix = prefill ? prompt_hidden : nullptr;
  ea.ids = (const int*)(ws + W.cur_ids);
  ea.hist = prefill ? (const int64_t*)(ws + W.raw_ids) : nullptr; ea.hist_ld = W.raw_ld;  // prefill: the n0 input columns
  ea.x = ws + W.x;
  ea.ctrl = ctrl;
  ea.B = B; ea.K = L.K; ea.V1 = L.V + 1; ea.H = H; ea.P = prefill ? P : 0; ea.n_cols = prefill ? s->n0 : 1;
  ea.pos_from_ctrl = prefill ? 0 : 1; ea.pos0 = 0; ea.prefix_len = P;
  // a ragged continuation's decode positions are per row; at prefill every row's column j sits at position P + j, as alone
  const int* shift = prefill ? nullptr : sample_args(s).shift;
  ea.shift = shift;
  if (int e = launch_embed(ea, c.dtype, st, pdl)) return e;
  s->launches++;

  // output_attentions / output_hidden_states (ptts_generate_set_probes): the prefill writes slot 0 when its window holds step 0,
  // a decode step finds its slot on the device (the graph is replayed for every step)
  const ProbeWindow* pw = active_probe(s);
  if (pw != nullptr && prefill && pw->first_step != 0) pw = nullptr;
  if (pw != nullptr && prefill && pw->self_attn != nullptr && pw->self_ld < q_len)
    return fail(PTTS_EINVAL, "probes: self_ld %lld is below the prefill's %d keys", (long long)pw->self_ld, q_len);
  const int64_t esz = es;
  auto probe_rows = [&](int entry, bool final_ln) -> int {
    if (pw == nullptr || pw->hidden == nullptr) return PTTS_OK;
    ProbeRowsArgs r{};
    r.x = ws + W.x; r.rows = M; r.H = H;
    if (final_ln) { r.ln_w = (const float*)(blob + L.final_ln_w); r.ln_b = (const float*)(blob + L.final_ln_b); }
    r.eps = c.layer_norm_eps;
    r.q_len = q_len; r.out_b = (int64_t)(L.L + 1) * q_len * H;   // [B][L+1][q][H]
    r.out = (char*)pw->hidden + (int64_t)entry * q_len * H * esz;
    r.ctrl = ctrl; r.n0 = s->n0; r.first_step = pw->first_step; r.n_steps = pw->n_steps; r.step_bytes = pw->hidden_step * esz;
    s->launches++;
    return launch_probe_rows(r, c.dtype, st);
  };
  auto probe_attn = [&](const AttnArgs& at, int layer) -> int {
    void* base = at.cross ? pw->cross_attn : pw->self_attn;
    if (base == nullptr) return PTTS_OK;
    AttnProbeArgs p{};
    p.q = at.q; p.ldq = at.ldq; p.q_col0 = at.q_col0;
    p.kcache = at.kcache; p.kv_b_stride = at.kv_b_stride; p.kv_h_stride = at.kv_h_stride; p.kv_b_div = at.kv_b_div;
    p.key_mask = at.key_mask; p.mask_len = at.mask_len; p.mask_ld = at.mask_ld;
    p.B = B; p.nh = L.nh; p.nkv = at.nkv; p.q_len = q_len; p.cross = at.cross;
    const int64_t ld = at.cross ? S : pw->self_ld;
    p.kv_len = at.cross ? S : q_len; p.pos0 = 0; p.kv_cap = at.cross ? S : (prefill ? q_len : W.Tmax);
    p.rope = at.rope; p.rope_cos = at.rope_cos; p.rope_sin = at.rope_sin; p.scale = at.scale;
    p.out_q = ld; p.out_h = (int64_t)q_len * ld; p.out_b = (int64_t)L.L * L.nh * p.out_h;   // [B][L][nh][q][ld]
    p.out = (char*)base + (int64_t)layer * L.nh * p.out_h * esz;
    p.ctrl = ctrl; p.n0 = s->n0; p.prefix = P; p.first_step = pw->first_step; p.n_steps = pw->n_steps;
    p.step_bytes = (at.cross ? pw->cross_step : pw->self_step) * esz;
    s->launches++;
    return launch_attention_probs(p, c.dtype, st);
  };
  if (int e = probe_rows(0, false)) return e;
  // return_token_timestamps (ptts_generate_set_alignment): decode steps only, after the attention whose keys hold the transcript
  const AlignWindow* aw = prefill ? nullptr : active_align(s);
  int align_done = 0;   // alignment heads written so far this step
  auto align_probe = [&](const AttnArgs& at, int layer) -> int {
    if (aw == nullptr || aw->layer_heads[layer] == 0 || (at.cross != 0) != (P == 0)) return PTTS_OK;
    AlignProbeArgs g{};
    g.q = at.q; g.ldq = at.ldq; g.q_col0 = at.q_col0;
    g.kcache = at.kcache; g.kv_b_stride = at.kv_b_stride; g.kv_h_stride = at.kv_h_stride; g.kv_b_div = at.kv_b_div;
    g.key_mask = at.key_mask; g.mask_ld = at.mask_ld;
    g.B = B; g.nh = L.nh; g.nkv = at.nkv; g.key0 = aw->key0; g.key_len = aw->key_len;
    g.heads = aw->heads; g.n_heads = aw->n_heads; g.layer = layer; g.layer_heads = aw->layer_heads[layer];
    g.weight = 1.0f / (float)aw->n_heads; g.accumulate = align_done > 0;
    g.rope = at.rope; g.rope_cos = at.rope_cos; g.rope_sin = at.rope_sin; g.scale = at.scale;
    g.out = aw->out; g.ctrl = ctrl; g.n0 = s->n0; g.prefix = P; g.first_row = aw->first_row; g.n_rows = aw->n_rows;
    align_done += g.layer_heads;
    s->launches++;
    return launch_alignment_probe(g, c.dtype, st);
  };

  // matrix `mat` of layer `layer` (decoder_matrix), with the LayerNorm in front of it where it has one.
  // plan_rows: the row count that picks the kernel (default Mrows); the GEMMs' per-row results do not depend on M otherwise
  auto lin = [&](const void* X, int64_t ldx, int mat, int layer, int epi, const void* R, void* Y, int64_t ldy, int Mrows,
                 int plan_rows = 0) -> int {
    const DecoderMatrix m = decoder_matrix(L, mat, layer);
    LinearArgs a{};
    a.X = X; a.ldx = ldx; a.W = blob + m.w; a.Y = Y; a.ldy = ldy; a.R = R; a.ldr = ldy;
    a.eps = c.layer_norm_eps;
    if (m.ln_w >= 0) {
      a.ln_w = (const float*)(blob + m.ln_w); a.ln_b = (const float*)(blob + m.ln_b);
      if (c.dtype == PTTS_BF16) { a.c1 = (const float*)(blob + m.c); a.c2 = a.c1 + m.N; }   // folded at load (ptts_decoder_finalize)
    }
    a.M = Mrows; a.N = m.N; a.K = m.K; a.Kc = (m.K > H && m.K % H == 0) ? H : m.K;
    a.epi = epi; a.act = c.activation; a.ctrl = ctrl;
    s->launches++;
    // the same matrix, row-major: M = B*(P+n0) or B*S rows are tensor-core work (wgmma, gemm_tc.cu)
    LinearArgs plan = a;
    if (plan_rows > 0) plan.M = plan_rows;
    if (prefill && m.rm >= 0 && linear_tc_supported(plan)) {
      if (a.c1 != nullptr) s->launches++;  // row statistics kernel
      return launch_linear_tc(a, blob + m.rm, (float*)(ws + W.row_stats), st);
    }
    return launch_linear(a, c.dtype, st, pdl, s->sm_count);
  };

  for (int i = 0; i < L.L; i++) {
    char* x = ws + W.x;
    if (prefill) {  // cross-attention K/V of the encoder states, once per generate() and description (:872-878)
      // the kernel is the one B * S rows take, so that the takes of a description get the bits B expanded rows would get (the
      // wgmma GEMM zero-fills the rows of a partial 128-row tile, also below 128 rows)
      if (int e = lin(enc_hidden, H, MAT_KV_CROSS, i, EPI_STORE, nullptr, ws + W.cross_tmp, L.ckv_rows, n_desc * S, B * S)) return e;
      if (int e = launch_cross_kv_relayout(ws + W.cross_tmp, ws + W.cross_kv + W.cross_layer_stride * i, n_desc, S, L.nckv, c.dtype, st)) return e;
      s->launches++;
    }
    if (int e = lin(x, H, MAT_QKV, i, EPI_STORE, nullptr, ws + W.qkv, L.qkv_rows, M)) return e;
    AttnArgs at{};
    at.q = ws + W.qkv; at.ldq = L.qkv_rows; at.q_col0 = 0;
    at.knew = ws + W.qkv; at.vnew = ws + W.qkv; at.ldkv = L.qkv_rows; at.k_col0 = L.nh * D; at.v_col0 = (L.nh + L.nkv) * D;
    char* kc = ws + W.self_kv + W.self_layer_stride * i;
    at.kcache = kc; at.vcache = kc + (int64_t)B * L.nkv * W.Tmax * D * es;
    at.kv_b_stride = (int64_t)L.nkv * W.Tmax * D; at.kv_h_stride = (int64_t)W.Tmax * D; at.kv_t_stride = D; at.kv_b_div = 1;
    at.out = ws + W.attn; at.ldo = H;
    at.key_mask = s->has_prompt_mask ? (const int*)(ws + W.prompt_mask) : nullptr; at.mask_len = P; at.mask_ld = P;
    at.ctrl = ctrl; at.B = B; at.nh = L.nh; at.nkv = L.nkv; at.q_len = q_len;
    at.past_from_ctrl = prefill ? 0 : 1; at.past_len = 0; at.prefix = P; at.shift = shift;
    at.cross = 0; at.kv_len = 0;
    at.rope = c.rope; at.rope_cos = blob + L.rope_cos; at.rope_sin = blob + L.rope_sin;
    at.kv_capacity = prefill ? q_len : W.Tmax;
    at.scale = 0.125f;  // head_dim ** -0.5, applied inside SDPA (quirk Q1)
    if (int e = launch_attention(at, c.dtype, st, pdl, true)) return e;
    s->launches++;
    if (pw != nullptr) { if (int e = probe_attn(at, i)) return e; }
    if (int e = align_probe(at, i)) return e;
    if (int e = lin(ws + W.attn, H, MAT_O, i, EPI_RESIDUAL, x, x, H, M)) return e;
    if (int e = lin(x, H, MAT_Q_CROSS, i, EPI_STORE, nullptr, ws + W.qc, H, M)) return e;
    AttnArgs ct = at;
    ct.q = ws + W.qc; ct.ldq = H; ct.q_col0 = 0;
    ct.knew = ct.vnew = nullptr;
    char* ck = ws + W.cross_kv + W.cross_layer_stride * i;
    ct.kcache = ck; ct.vcache = ck + (int64_t)n_desc * L.nckv * S * D * es;   // item-major: K [B/takes][nckv][S][64] | V [...]
    ct.kv_b_stride = (int64_t)L.nckv * S * D; ct.kv_h_stride = (int64_t)S * D; ct.kv_t_stride = D; ct.kv_b_div = W.takes;
    ct.key_mask = s->has_enc_mask ? (const int*)(ws + W.enc_mask) : nullptr; ct.mask_len = S; ct.mask_ld = S;
    ct.nkv = L.nckv; ct.cross = 1; ct.kv_len = S; ct.kv_capacity = S;
    if (int e = launch_attention(ct, c.dtype, st, pdl, true)) return e;
    s->launches++;
    if (pw != nullptr) { if (int e = probe_attn(ct, i)) return e; }
    if (int e = align_probe(ct, i)) return e;
    if (int e = lin(ws + W.attn, H, MAT_O_CROSS, i, EPI_RESIDUAL, x, x, H, M)) return e;
    if (int e = lin(x, H, MAT_FC1, i, EPI_ACT, nullptr, ws + W.hbuf, L.F, M)) return e;
    if (int e = lin(ws + W.hbuf, L.F, MAT_FC2, i, EPI_RESIDUAL, x, x, H, M)) return e;
    if (int e = probe_rows(i + 1, i == L.L - 1)) return e;   // entry L: the final LayerNorm of the last layer's output
  }
  if (!heads) return PTTS_OK;
  // final LayerNorm + K lm heads on the last position of every batch row -> f32 logits [B, K*V] == [B*K, V]
  if (prefill && s->ragged) {
    // a ragged continuation's row b ends at its own last input column, row P + n0_b - 1 = q_len - 1 - shift[b].  Its padded
    // columns past it were embedded and wrote K/V into cache slots >= P + n0_b, which no query has seen: the causal mask keeps
    // the row's own queries off them, and decode step t appends slot P + n0_b + t before its query reads keys up to it.
    if (int e = launch_gather_rows(ws + W.x, H, q_len - 1, q_len, sample_args(s).shift, ws + W.hidden, B, H, c.dtype, st)) return e;
    s->launches++;
    return lin(ws + W.hidden, H, MAT_HEADS, 0, EPI_F32, nullptr, ws + W.logits, (int64_t)L.K * L.V, B);
  }
  const char* xlast = ws + W.x + (int64_t)(q_len - 1) * H * es;
  return lin(xlast, (int64_t)q_len * H, MAT_HEADS, 0, EPI_F32, nullptr, ws + W.logits, (int64_t)L.K * L.V, B);
}

int ptts_prefill(ptts_session* s, const void* prompt_hidden, const int64_t* prompt_mask, const void* enc_hidden,
                 const int64_t* enc_mask, void* stream) {
  PTTS_REQUIRE(s && enc_hidden, "null argument");
  if (!s->begun) return fail(PTTS_ESTATE, "ptts_prefill called before ptts_generate_begin");
  PTTS_REQUIRE(s->W.P == 0 || prompt_hidden, "prefill: prompt_hidden is required when P > 0");
  cudaStream_t st = (cudaStream_t)stream;
  s->has_prompt_mask = (prompt_mask != nullptr && s->W.P > 0);
  s->has_enc_mask = (enc_mask != nullptr);
  if (s->has_prompt_mask) { if (int e = launch_mask_convert(prompt_mask, s->W.B * s->W.P, (int*)(s->ws + s->W.prompt_mask), st)) return e; }
  if (s->has_enc_mask) { if (int e = launch_mask_convert(enc_mask, s->W.B / s->W.takes * s->W.S, (int*)(s->ws + s->W.enc_mask), st)) return e; }
  if (int e = run_forward(s, st, true, prompt_hidden, enc_hidden)) return e;
  s->prefilled = true;
  s->sampled = 0;
  s->decoded = false;
  s->path = choose_decode_path(s);
  // mask presence is baked into the captured graph: re-capture if it changed
  drop_graph(s);
  return PTTS_OK;
}

// ---- teacher-forced scoring --------------------------------------------------------------------
int ptts_lm_heads_rowmajor_bytes(const ptts_decoder_config* cfg, int64_t* out_bytes) {
  PTTS_REQUIRE(cfg && out_bytes, "null argument");
  if (int e = validate_config(*cfg)) return e;
  PTTS_REQUIRE(cfg->dtype == PTTS_BF16, "lm heads row-major copy: only bf16 models score on the fused kernel");
  *out_bytes = (int64_t)cfg->num_codebooks * cfg->vocab_size * cfg->hidden_size * 2;
  return PTTS_OK;
}

int ptts_lm_heads_rowmajor_pack(const ptts_decoder_config* cfg, const void* blob, void* heads_rm, void* stream) {
  PTTS_REQUIRE(cfg && blob && heads_rm, "null argument");
  if (int e = validate_config(*cfg)) return e;
  PTTS_REQUIRE(cfg->dtype == PTTS_BF16, "lm heads row-major copy: only bf16 models score on the fused kernel");
  const DecoderLayout L = make_layout(*cfg);
  return unpack_fragments((const char*)blob + L.heads, heads_rm, (int64_t)L.K * L.V, L.H, (cudaStream_t)stream);
}

// The scoring heads over the residual stream x [B][P+T][H] (ptts_score after its forward pass, and ptts_op_score): fused, the
// label-row gather and the heads + cross-entropy kernel; unfused, the decoder's heads GEMM over the B rows of one frame at a time
// into logits_scratch [B*K][V], then score_rows_kernel; then the per-codebook reduce when codebook_sums is given.
static int score_heads(const ptts_decoder_config& c, const DecoderLayout& L, const char* blob, const void* heads_rm, const char* x,
                       int B, int P, int T, const int64_t* labels, const int64_t* dec_ids, bool fused, float* token_nll,
                       float* out_logits, float* codebook_sums, void* xs_scratch, float* row_stats, float* logits_scratch,
                       int sm_count, int64_t* launches, cudaStream_t st) {
  ScoreArgs a{};
  a.labels = labels; a.dec_ids = dec_ids; a.token_nll = token_nll;
  a.M = B * T; a.B = B; a.T = T; a.K = L.K; a.V = L.V; a.H = L.H;
  a.bos = c.bos_token_id; a.eos = c.eos_token_id;
  const int q_len = P + T;
  const DecoderMatrix hm = decoder_matrix(L, MAT_HEADS, 0);
  if (fused) {
    a.c1 = (const float*)(blob + hm.c); a.c2 = a.c1 + hm.N;
    *launches += 2;
    if (int e = launch_score_fused(a, x, P, c.layer_norm_eps, xs_scratch, row_stats, heads_rm, st)) return e;
  } else {
    for (int t = 0; t < T; t++) {
      LinearArgs h{};
      h.X = x + (int64_t)(P + t) * L.H * L.es; h.ldx = (int64_t)q_len * L.H;
      h.W = blob + hm.w; h.Y = logits_scratch; h.ldy = hm.N; h.ldr = h.ldy;
      h.ln_w = (const float*)(blob + hm.ln_w); h.ln_b = (const float*)(blob + hm.ln_b); h.eps = c.layer_norm_eps;
      if (c.dtype == PTTS_BF16) { h.c1 = (const float*)(blob + hm.c); h.c2 = h.c1 + hm.N; }
      h.M = B; h.N = hm.N; h.K = hm.K; h.Kc = hm.K;
      h.epi = EPI_F32; h.act = c.activation;
      if (int e = launch_linear(h, c.dtype, st, false, sm_count)) return e;
      if (int e = launch_score_rows(a, logits_scratch, t, out_logits, st)) return e;
      *launches += 2;
    }
  }
  if (codebook_sums != nullptr) {
    (*launches)++;
    if (int e = launch_score_reduce(a, codebook_sums, st)) return e;
  }
  return PTTS_OK;
}

int ptts_score(ptts_session* s, const void* prompt_hidden, const int64_t* prompt_mask, const void* enc_hidden, const int64_t* enc_mask,
               const int64_t* dec_ids, const int64_t* labels, int32_t T, const void* heads_rm, float* out_token_nll, float* out_logits,
               float* out_codebook_sums, void* stream) {
  PTTS_REQUIRE(s && enc_hidden && dec_ids, "null argument");
  const ptts_decoder_config& c = s->cfg;
  const DecoderLayout& L = s->L;
  const WorkspaceLayout& W = s->W;
  PTTS_REQUIRE(T >= 1 && T <= W.max_input, "score: %d decoder input columns, the session takes 1 .. %d", T, W.max_input);
  PTTS_REQUIRE(W.P == 0 || prompt_hidden, "score: prompt_hidden is required when P > 0");
  PTTS_REQUIRE(labels ? (out_token_nll != nullptr) : (out_logits != nullptr && out_codebook_sums == nullptr),
               "score: labels need out_token_nll; without labels only out_logits can be filled");
  const bool fused = (c.dtype == PTTS_BF16 && out_logits == nullptr);
  PTTS_REQUIRE(!fused || heads_rm, "score: the fused bf16 path needs the row-major heads (ptts_lm_heads_rowmajor_pack)");
  PTTS_REQUIRE(!fused || score_fused_supported(L.H, L.V), "score: hidden_size %d / vocab_size %d are outside the fused kernel", L.H, L.V);
  cudaStream_t st = (cudaStream_t)stream;
  // the decoder input goes into the history as given: it is already delayed (no ptts_generate_begin_ids)
  PTTS_CHECK_CUDA(cudaMemcpy2DAsync(s->ws + W.raw_ids, W.raw_ld * 8, dec_ids, (size_t)T * 8, (size_t)T * 8, W.BK, cudaMemcpyDeviceToDevice, st));
  s->has_prompt_mask = (prompt_mask != nullptr && W.P > 0);
  s->has_enc_mask = (enc_mask != nullptr);
  if (s->has_prompt_mask) { if (int e = launch_mask_convert(prompt_mask, W.B * W.P, (int*)(s->ws + W.prompt_mask), st)) return e; }
  if (s->has_enc_mask) { if (int e = launch_mask_convert(enc_mask, W.B / W.takes * W.S, (int*)(s->ws + W.enc_mask), st)) return e; }
  s->n0 = T;
  s->ragged = s->slots = false;
  s->begun = s->prefilled = false;  // the caches now hold this call's positions: a generation has to begin again
  if (int e = run_forward(s, st, true, prompt_hidden, enc_hidden, false)) return e;
  return score_heads(c, L, s->blob, heads_rm, s->ws + W.x, W.B, W.P, T, labels, dec_ids, fused, out_token_nll, out_logits,
                     out_codebook_sums, s->ws + W.qc, (float*)(s->ws + W.row_stats), (float*)(s->ws + W.logits), s->sm_count,
                     &s->launches, st);
}

int ptts_decode_forward(ptts_session* s, void* stream) {
  PTTS_REQUIRE(s, "null argument");
  if (!s->prefilled) return fail(PTTS_ESTATE, "ptts_decode_forward called before ptts_prefill");
  cudaStream_t st = (cudaStream_t)stream;
  s->decoded = true;
  StepParams p = s->sp;
  p.do_sample_phase = 0;
  switch (decode_path(s)) {
    case DECODE_CLUSTER: s->launches++; return launch_decode_step_cluster(p, st);
    case DECODE_STEP: s->launches++; return launch_decode_step(p, s->sm_count, st);
    case DECODE_MULTI_KERNEL: break;
  }
  return run_forward(s, st, false, nullptr, nullptr);
}

int ptts_sample(ptts_session* s, const int64_t* forced_tokens, void* stream) {
  PTTS_REQUIRE(s, "null argument");
  if (!s->prefilled) return fail(PTTS_ESTATE, "ptts_sample called before ptts_prefill");
  s->launches++;
  s->sampled++;
  return launch_sample(sample_args(s), forced_tokens, (cudaStream_t)stream, false, sampler_ext(s), active_out(s), active_lext(s),
                       slot_keys(s), slot_max_lens(s));
}

int ptts_decode_steps(ptts_session* s, int32_t n_steps, void* stream) {
  PTTS_REQUIRE(s && n_steps >= 0, "bad argument");
  if (!s->prefilled) return fail(PTTS_ESTATE, "ptts_decode_steps called before ptts_prefill");
  cudaStream_t st = (cudaStream_t)stream;
  if (n_steps > 0) s->decoded = true;
  const ptts_sampling_ext* ext = sampler_ext(s);
  const SampleOut* out = active_out(s);
  const ptts_logits_ext* lext = active_lext(s);
  const DecodePath path = decode_path(s);
  if (ext != nullptr && path != DECODE_MULTI_KERNEL) {
    // an EXT stage is active or the outputs are set: the step kernel stops at the logits and the EXT sampler follows, token by
    // token; both return at once after the last token
    StepParams p = s->sp;
    p.do_sample_phase = 0;
    for (int i = 0; i < n_steps; i++) {
      const int e = path == DECODE_CLUSTER ? launch_decode_step_cluster(p, st) : launch_decode_step(p, s->sm_count, st);
      if (e) return e;
      if (int e2 = launch_sample(sample_args(s), nullptr, st, false, ext, out, lext, slot_keys(s), slot_max_lens(s))) return e2;
    }
    s->launches += 2 * (int64_t)n_steps;
    return PTTS_OK;
  }
  switch (path) {
    case DECODE_CLUSTER: {  // the kernel loops over tokens itself: up to PTTS_STEPS_PER_LAUNCH (default 64) per launch
      const char* env = getenv("PTTS_STEPS_PER_LAUNCH");   // (read per call: tests compare 1 against the default)
      const int per_launch = env ? (atoi(env) < 1 ? 1 : atoi(env)) : 64;
      for (int done = 0; done < n_steps;) {
        const int m = (n_steps - done < per_launch) ? n_steps - done : per_launch;
        s->sp.n_steps = m;
        const int e = launch_decode_step_cluster(s->sp, st);
        s->sp.n_steps = 1;
        if (e) return e;
        done += m;
        s->launches += 1;
      }
      return PTTS_OK;
    }
    case DECODE_STEP:  // one persistent kernel per token: nothing to gain from a graph
      for (int i = 0; i < n_steps; i++)
        if (int e = launch_decode_step(s->sp, s->sm_count, st)) return e;
      s->launches += n_steps;
      return PTTS_OK;
    case DECODE_MULTI_KERNEL: break;
  }
  if (!s->graph_ready) {
    if (!s->cap_stream) PTTS_CHECK_CUDA(cudaStreamCreateWithFlags(&s->cap_stream, cudaStreamNonBlocking));
    const int64_t before = s->launches;
    PTTS_CHECK_CUDA(cudaStreamBeginCapture(s->cap_stream, cudaStreamCaptureModeThreadLocal));
    int e = run_forward(s, s->cap_stream, false, nullptr, nullptr);
    if (!e) { s->launches++; e = launch_sample(sample_args(s), nullptr, s->cap_stream, true, ext, out, lext, slot_keys(s), slot_max_lens(s)); }
    cudaGraph_t graph = nullptr;
    cudaError_t ce = cudaStreamEndCapture(s->cap_stream, &graph);
    s->graph_launches = s->launches - before;   // embed + 8 kernels per layer + heads + sample (+ the probe kernels)
    s->launches = before;
    if (e) { if (graph) cudaGraphDestroy(graph); return e; }
    if (ce != cudaSuccess) return fail(PTTS_ECUDA, "graph capture failed: %s", cudaGetErrorString(ce));
    ce = cudaGraphInstantiate(&s->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) return fail(PTTS_ECUDA, "graph instantiate failed: %s", cudaGetErrorString(ce));
    s->graph_ready = true;
  }
  for (int i = 0; i < n_steps; i++) PTTS_CHECK_CUDA(cudaGraphLaunch(s->exec, st));
  s->launches += s->graph_launches * n_steps;
  return PTTS_OK;
}

// ---- continuous batching ------------------------------------------------------------------------
int ptts_session_import_rows(ptts_session* dst, const ptts_session* src, const int32_t* src_rows, const int32_t* dst_rows, int32_t n,
                             void* stream) {
  PTTS_REQUIRE(dst && src && (n == 0 || (src_rows && dst_rows)) && n >= 0, "bad argument");
  if (!src->prefilled || !dst->prefilled) return fail(PTTS_ESTATE, "import_rows: both sessions must have run ptts_prefill");
  PTTS_REQUIRE(dst != src, "import_rows: the source and the destination are one session");
  PTTS_REQUIRE(memcmp(&src->cfg, &dst->cfg, sizeof(src->cfg)) == 0 && src->blob == dst->blob, "import_rows: the sessions run different models");
  PTTS_REQUIRE(src->W.P == dst->W.P && src->W.S == dst->W.S, "import_rows: P and S must match (source %d, %d; destination %d, %d)",
               src->W.P, src->W.S, dst->W.P, dst->W.S);
  PTTS_REQUIRE(src->W.takes == 1 && dst->W.takes == 1, "import_rows: sessions with takes > 1 share cross K/V between rows");
  PTTS_REQUIRE(src->has_prompt_mask == dst->has_prompt_mask && src->has_enc_mask == dst->has_enc_mask,
               "import_rows: both sessions must have been prefilled with the same masks given (or both without)");
  PTTS_REQUIRE(!src->ragged && src->n0 == 1, "import_rows: the source rows must start from the BOS column (a uniform generation)");
  // the cache holds positions [0, P + 1) and the history columns [0, 2) only then
  PTTS_REQUIRE(src->sampled == 1 && !src->decoded, "import_rows: the source must have run ptts_prefill and exactly one ptts_sample "
               "since (%d samples%s)", src->sampled, src->decoded ? " and decode steps" : "");
  const int kv_len = src->W.P + src->n0;
  PTTS_REQUIRE(kv_len <= dst->W.Tmax, "import_rows: %d cache positions do not fit the destination's %d", kv_len, dst->W.Tmax);
  RowImportArgs a{};
  RowRegion tmp[kMaxRowRegions];
  a.n_regions = row_regions(src->cfg, src->W, kv_len, a.src);
  PTTS_REQUIRE(row_regions(dst->cfg, dst->W, kv_len, tmp) == a.n_regions, "import_rows: the sessions hold different per-row state "
               "(create both with the same max_input_len class: 1, or >= 2)");
  for (int r = 0; r < a.n_regions; r++) a.dst[r] = tmp[r];
  a.src_ws = src->ws; a.dst_ws = dst->ws; a.K = src->cfg.num_codebooks;
  a.src_ctrl = (const Ctrl*)(src->ws + src->W.ctrl); a.dst_ctrl = (const Ctrl*)(dst->ws + dst->W.ctrl);
  std::vector<char> taken(dst->W.B, 0);
  for (int i = 0; i < n; i++) {
    PTTS_REQUIRE(src_rows[i] >= 0 && src_rows[i] < src->W.B, "import_rows: source row %d outside [0, %d)", src_rows[i], src->W.B);
    PTTS_REQUIRE(dst_rows[i] >= 0 && dst_rows[i] < dst->W.B, "import_rows: destination row %d outside [0, %d)", dst_rows[i], dst->W.B);
    PTTS_REQUIRE(!taken[dst_rows[i]], "import_rows: destination row %d is listed twice", dst_rows[i]);
    taken[dst_rows[i]] = 1;
  }
  for (int i0 = 0; i0 < n; i0 += kMaxImportRows) {
    const int m = n - i0 < kMaxImportRows ? n - i0 : kMaxImportRows;
    for (int i = 0; i < m; i++) { a.src_row[i] = src_rows[i0 + i]; a.dst_row[i] = dst_rows[i0 + i]; }
    if (int e = launch_import_rows(a, m, (cudaStream_t)stream)) return e;
    dst->launches++;
  }
  return PTTS_OK;
}

int ptts_generate_set_slots(ptts_session* s, int32_t cur_len, const int32_t* row_shift, const int32_t* row_key, void* stream) {
  return ptts_generate_set_slots2(s, cur_len, row_shift, row_key, nullptr, stream);
}

int ptts_generate_set_slots2(ptts_session* s, int32_t cur_len, const int32_t* row_shift, const int32_t* row_key,
                             const int32_t* row_max_length, void* stream) {
  PTTS_REQUIRE(s && row_shift && row_key, "null argument");
  if (!s->prefilled) return fail(PTTS_ESTATE, "set_slots called before ptts_prefill");
  const WorkspaceLayout& W = s->W;
  PTTS_REQUIRE(W.row_shift >= 0, "set_slots: the session has no per-row offsets (create it with max_input_len >= 2)");
  PTTS_REQUIRE(W.takes == 1, "set_slots: a session with takes > 1 shares cross K/V between rows");
  PTTS_REQUIRE(s->n0 == 1 && (!s->ragged || s->slots), "set_slots: slot mode takes requests that start from the BOS column");
  PTTS_REQUIRE(active_probe(s) == nullptr && active_align(s) == nullptr && active_out(s) == nullptr,
               "set_slots: the probe and per-step output windows count one batch step, not a slot's column");
  const ptts_logits_ext& lx = s->lext;
  PTTS_REQUIRE(lx.forced_eos_token_id < 0 && lx.decay == nullptr && lx.begin_suppress == nullptr,
               "set_slots: forced_eos_token_id, the decay penalty and begin_suppress_tokens count from one batch column");
  PTTS_REQUIRE(cur_len >= 1 && cur_len < W.raw_ld, "set_slots: cur_len %d outside [1, %lld)", cur_len, (long long)W.raw_ld);
  for (int b = 0; b < W.B; b++) {
    PTTS_REQUIRE(row_shift[b] >= 0 && row_shift[b] < cur_len, "set_slots: row_shift[%d] = %d outside [0, cur_len = %d)", b, row_shift[b], cur_len);
    PTTS_REQUIRE(row_key[b] >= 0, "set_slots: row_key[%d] = %d is negative", b, row_key[b]);
  }
  // a row's first column was drawn under gen.max_length before slot mode: a limit of at least 2K - 1 (and 2) is on the same side
  // of the delay pattern's gate and neither stops nor pads that column, so the row holds what its own limit gives it
  const int lo = 2 * s->cfg.num_codebooks - 1 > 2 ? 2 * s->cfg.num_codebooks - 1 : 2, hi = s->gen.max_length;
  std::vector<int32_t> lims(W.B, hi);
  if (row_max_length != nullptr)
    for (int b = 0; b < W.B; b++) {
      PTTS_REQUIRE(row_max_length[b] >= lo && row_max_length[b] <= hi, "set_slots: row_max_length[%d] = %d outside [%d, max_length = %d]",
                   b, row_max_length[b], lo, hi);
      lims[b] = row_max_length[b];
    }
  if (int e = launch_set_slots((Ctrl*)(s->ws + W.ctrl), cur_len, (int*)(s->ws + W.row_shift), (int*)(s->ws + W.row_key),
                               (int*)(s->ws + W.row_max_len), row_shift, row_key, lims.data(), W.B, (cudaStream_t)stream)) return e;
  s->launches += (W.B + kMaxSlotRows - 1) / kMaxSlotRows;
  if (!s->slots) {   // the decode kernels switch to their ragged instantiations (set up anew) and the sampler to slot mode
    s->ragged = s->slots = true;
    s->path = choose_decode_path(s);
    drop_graph(s);
  }
  return PTTS_OK;
}

int ptts_align_dtw(const float* alignment, int32_t B, int32_t T, int32_t P, const int32_t* n_frames, const int32_t* key_mask,
                   float* filtered, uint8_t* trace, int32_t* jumps, void* stream) {
  PTTS_REQUIRE(alignment && n_frames && filtered && trace && jumps, "null argument");
  return launch_align_dtw(alignment, B, T, P, n_frames, key_mask, filtered, trace, jumps, (cudaStream_t)stream);
}

int ptts_session_logits(ptts_session* s, float** out) { PTTS_REQUIRE(s && out, "null"); *out = (float*)(s->ws + s->W.logits); return PTTS_OK; }
int ptts_session_scores(ptts_session* s, float** out) { PTTS_REQUIRE(s && out, "null"); *out = (float*)(s->ws + s->W.scores); return PTTS_OK; }
int ptts_session_raw_ids(ptts_session* s, int64_t** out, int32_t* ld) {
  PTTS_REQUIRE(s && out && ld, "null");
  *out = (int64_t*)(s->ws + s->W.raw_ids);
  *ld = (int32_t)s->W.raw_ld;
  return PTTS_OK;
}
int ptts_session_eos_seen(ptts_session* s, int32_t** out) {
  PTTS_REQUIRE(s && out, "null");
  *out = (int32_t*)(s->ws + s->W.eos_seen);
  return PTTS_OK;
}
int ptts_session_state(ptts_session* s, int32_t** out) { PTTS_REQUIRE(s && out, "null"); *out = (int32_t*)(s->ws + s->W.ctrl); return PTTS_OK; }
// Debug / profiling aid: CTA 0 of the fused step kernel writes clock64() stamps per phase into `buf`
// (device int64 [(8L+2)*8]); pass NULL to switch it off.  Only the next launches are affected.
int ptts_session_set_profile(ptts_session* s, void* buf) {
  PTTS_REQUIRE(s, "null");
  s->prof = (long long*)buf;
  s->sp.prof = s->prof;
  return PTTS_OK;
}
int ptts_session_fused(ptts_session* s, int32_t* out) { PTTS_REQUIRE(s && out, "null"); *out = s->path; return PTTS_OK; }
int ptts_session_launches(ptts_session* s, int64_t* out) { PTTS_REQUIRE(s && out, "null"); *out = s->launches; return PTTS_OK; }

// ---- stand-alone operators ----------------------------------------------------------------------
int ptts_delay_build(const int64_t* input_ids, int32_t BK, int32_t seq_len, int32_t num_codebooks, int64_t bos, int64_t pad,
                     int32_t max_length, int64_t* pattern_mask, void* stream) {
  PTTS_REQUIRE(input_ids && pattern_mask, "null argument");
  PTTS_REQUIRE(num_codebooks > 0 && BK > 0 && BK % num_codebooks == 0 && seq_len > 0 && max_length > 0, "delay_build: bad shape");
  return launch_delay_build(input_ids, BK, seq_len, num_codebooks, bos, pad, max_length, pattern_mask, (cudaStream_t)stream);
}
int ptts_delay_apply(const int64_t* input_ids, int32_t BK, int32_t seq_len, int64_t ld_ids, const int64_t* pattern_mask,
                     int64_t ld_mask, int64_t* out, void* stream) {
  PTTS_REQUIRE(input_ids && pattern_mask && out, "null argument");
  PTTS_REQUIRE(BK > 0 && seq_len > 0 && ld_mask >= seq_len && ld_ids >= seq_len, "delay_apply: mask shorter than ids");
  return launch_delay_apply(input_ids, BK, seq_len, ld_ids, pattern_mask, ld_mask, out, (cudaStream_t)stream);
}
int ptts_logits_processor(const int64_t* input_ids, int32_t BK, int32_t seq_len, int64_t ld_ids, float* scores, int32_t V,
                          int64_t eos, int32_t num_codebooks, int64_t* first_unfinished, void* stream) {
  PTTS_REQUIRE(input_ids && scores && first_unfinished, "null argument");
  return launch_logits_processor(input_ids, BK, seq_len, ld_ids, scores, V, eos, num_codebooks, first_unfinished, (cudaStream_t)stream);
}

int ptts_op_sample_phase(ptts_session* s, int32_t n_ctas, void* stream) {
  PTTS_REQUIRE(s, "null argument");
  if (!s->prefilled) return fail(PTTS_ESTATE, "ptts_op_sample_phase called before ptts_prefill");
  PTTS_REQUIRE(sampler_ext(s) == nullptr, "op_sample_phase: the step kernels' sampling phase has no ptts_sampling_ext or "
                                          "ptts_logits_ext stages and records no per-step outputs; switch them off first");
  s->launches++;
  s->sampled++;
  return launch_sample_phase(sample_args(s), n_ctas, (cudaStream_t)stream);
}

int ptts_op_linear2(const ptts_decoder_config* cfg, const void* blob, int32_t tensor_id, int32_t index, const void* x, int32_t M,
                    int32_t use_ln, int32_t epilogue, const void* residual, void* y, int32_t path, float* row_stats, void* stream) {
  PTTS_REQUIRE(cfg && blob && x && y, "null argument");
  PTTS_REQUIRE(path == 0 || path == 1, "op_linear: path is 0 (decode GEMM) or 1 (wgmma prefill GEMM), got %d", path);
  PTTS_REQUIRE(M > 0, "op_linear: M must be positive, got %d", M);
  if (int e = validate_config(*cfg)) return e;
  const DecoderLayout L = make_layout(*cfg);
  MatSlot ms;
  PTTS_REQUIRE(matrix_slot(L, tensor_id, index, &ms), "op_linear: tensor %d is not a matrix", tensor_id);
  const DecoderMatrix& m = ms.m;
  const char* bl = (const char*)blob;
  LinearArgs a{};
  a.X = x; a.ldx = m.K; a.W = bl + m.w; a.Y = y; a.ldy = m.N; a.R = residual; a.ldr = m.N;
  if (use_ln) {
    PTTS_REQUIRE(m.K == L.H, "op_linear: LayerNorm needs K == hidden_size");
    PTTS_REQUIRE(m.ln_w >= 0, "op_linear: tensor %d has no LayerNorm in front", tensor_id);
    a.ln_w = (const float*)(bl + m.ln_w);
    a.ln_b = (const float*)(bl + m.ln_b);
    if (cfg->dtype == PTTS_BF16) { a.c1 = (const float*)(bl + m.c); a.c2 = a.c1 + m.N; }
  }
  a.eps = cfg->layer_norm_eps;
  a.M = M; a.N = m.N; a.K = m.K; a.Kc = (m.K > L.H && m.K % L.H == 0) ? L.H : m.K;
  a.epi = epilogue; a.act = cfg->activation; a.ctrl = nullptr;
  PTTS_REQUIRE(epilogue >= 0 && epilogue <= 3, "op_linear: bad epilogue");
  PTTS_REQUIRE(epilogue != EPI_RESIDUAL || residual, "op_linear: residual required");
  if (path == 1) {  // the prefill's rule: bf16, linear_tc_supported, a row-major copy
    PTTS_REQUIRE(cfg->dtype == PTTS_BF16 && linear_tc_supported(a), "op_linear: the wgmma GEMM does not take this problem (dtype %d, M %d, N %d, K %d, epilogue %d)",
                 cfg->dtype, M, m.N, m.K, epilogue);
    PTTS_REQUIRE(m.rm >= 0, "op_linear: tensor %d has no row-major copy for the wgmma GEMM", tensor_id);
    PTTS_REQUIRE(a.c1 == nullptr || row_stats, "op_linear: row_stats scratch required with LayerNorm");
    return launch_linear_tc(a, bl + m.rm, row_stats, (cudaStream_t)stream);
  }
  int sm = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, dev);
  return launch_linear(a, cfg->dtype, (cudaStream_t)stream, false, sm);
}

int ptts_op_linear(const ptts_decoder_config* cfg, const void* blob, int32_t tensor_id, int32_t index, const void* x, int32_t M,
                   int32_t use_ln, int32_t epilogue, const void* residual, void* y, void* stream) {
  return ptts_op_linear2(cfg, blob, tensor_id, index, x, M, use_ln, epilogue, residual, y, 0, nullptr, stream);
}

int ptts_op_score(const ptts_decoder_config* cfg, const void* blob, const void* heads_rm, const void* x, int32_t B, int32_t P,
                  int32_t T, const int64_t* labels, const int64_t* dec_ids, int32_t path, float* token_nll, float* out_logits,
                  float* codebook_sums, void* xs_scratch, float* row_stats, float* logits_scratch, void* stream) {
  PTTS_REQUIRE(cfg && blob && x && dec_ids, "null argument");
  PTTS_REQUIRE(path == 0 || path == 1, "op_score: path is 0 (heads GEMM + score_rows) or 1 (fused heads + cross-entropy), got %d", path);
  PTTS_REQUIRE(B >= 1 && P >= 0 && T >= 1, "op_score: needs B >= 1, P >= 0, T >= 1, got B %d P %d T %d", B, P, T);
  if (int e = validate_config(*cfg)) return e;
  const DecoderLayout L = make_layout(*cfg);
  PTTS_REQUIRE(labels ? (token_nll != nullptr) : (out_logits != nullptr && codebook_sums == nullptr),
               "op_score: labels need token_nll; without labels only out_logits can be filled");
  if (path == 1) {  // the rule of ptts_score: bf16, no logits wanted, a shape the fused kernel takes, the row-major heads
    PTTS_REQUIRE(cfg->dtype == PTTS_BF16, "op_score: the fused kernel is bf16 only");
    PTTS_REQUIRE(labels && out_logits == nullptr, "op_score: the fused kernel needs labels and writes no logits");
    PTTS_REQUIRE(score_fused_supported(L.H, L.V), "op_score: hidden_size %d / vocab_size %d are outside the fused kernel", L.H, L.V);
    PTTS_REQUIRE(heads_rm && xs_scratch && row_stats, "op_score: the fused kernel needs heads_rm, xs_scratch [B*T][H] and row_stats [B*T][2]");
  } else {
    PTTS_REQUIRE(logits_scratch, "op_score: the heads GEMM needs logits_scratch [B*K][V]");
  }
  int sm = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, dev);
  int64_t launches = 0;
  return score_heads(*cfg, L, (const char*)blob, heads_rm, (const char*)x, B, P, T, labels, dec_ids, path == 1, token_nll, out_logits,
                     codebook_sums, xs_scratch, row_stats, logits_scratch, sm, &launches, (cudaStream_t)stream);
}

int ptts_op_attention(int32_t dtype, int32_t B, int32_t nh, int32_t nkv, int32_t q_len, int32_t past_len, int32_t cross,
                      int32_t kv_len, int32_t capacity, int32_t rope, const void* rope_cos, const void* rope_sin, const void* qkv,
                      void* kcache, void* vcache, const int32_t* key_mask, int32_t mask_len, int32_t prefill_sweep, void* out,
                      void* stream) {
  PTTS_REQUIRE(qkv && kcache && vcache && out, "null argument");
  PTTS_REQUIRE(dtype == PTTS_BF16 || dtype == PTTS_F32, "op_attention: dtype must be bf16 or f32");
  PTTS_REQUIRE(B > 0 && nh > 0 && nkv > 0 && nh % nkv == 0 && q_len > 0 && past_len >= 0, "op_attention: bad shape");
  PTTS_REQUIRE(cross ? (kv_len > 0 && kv_len <= capacity) : (past_len + q_len <= capacity),
               "op_attention: %d keys do not fit a cache of %d positions", cross ? kv_len : past_len + q_len, capacity);
  PTTS_REQUIRE(!rope || (rope_cos && rope_sin), "op_attention: rope needs both tables");
  PTTS_REQUIRE(mask_len >= 0 && (key_mask || mask_len == 0), "op_attention: bad key mask");
  PTTS_REQUIRE(prefill_sweep == 0 || prefill_sweep == 1, "op_attention: prefill_sweep is 0 (product choice) or 1 (attention_item)");
  const int D = PTTS_HEAD_DIM;
  AttnArgs a{};
  if (cross) {  // q [B*q_len, nh*64]
    a.q = qkv; a.ldq = (int64_t)nh * D;
  } else {      // fused projections [B*q_len, (nh + 2 nkv)*64]: q | k | v, as run_forward's qkv matrix
    a.q = a.knew = a.vnew = qkv;
    a.ldq = a.ldkv = (int64_t)(nh + 2 * nkv) * D; a.k_col0 = nh * D; a.v_col0 = (nh + nkv) * D;
  }
  a.kcache = kcache; a.vcache = vcache;
  a.kv_b_stride = (int64_t)nkv * capacity * D; a.kv_h_stride = (int64_t)capacity * D; a.kv_t_stride = D; a.kv_b_div = 1;
  a.out = out; a.ldo = (int64_t)nh * D;
  a.key_mask = key_mask; a.mask_len = mask_len; a.mask_ld = mask_len;
  a.B = B; a.nh = nh; a.nkv = nkv; a.q_len = q_len;
  a.past_len = past_len; a.cross = cross ? 1 : 0; a.kv_len = cross ? kv_len : 0;
  a.rope = rope; a.rope_cos = rope_cos; a.rope_sin = rope_sin;
  a.kv_capacity = cross ? kv_len : past_len + q_len;   // keys per query at most (attention_item's score buffer)
  a.scale = 0.125f;
  return launch_attention(a, dtype, (cudaStream_t)stream, false, prefill_sweep == 0);
}

int ptts_op_attention_probs(int32_t dtype, int32_t B, int32_t nh, int32_t nkv, int32_t q_len, int32_t past_len, int32_t cross,
                            int32_t kv_len, int32_t capacity, int32_t rope, const void* rope_cos, const void* rope_sin, const void* q,
                            int64_t ldq, const void* kcache, const int32_t* key_mask, int32_t mask_len, void* out, void* stream) {
  PTTS_REQUIRE(q && kcache && out, "null argument");
  PTTS_REQUIRE(dtype == PTTS_BF16 || dtype == PTTS_F32, "op_attention_probs: dtype must be bf16 or f32");
  PTTS_REQUIRE(B > 0 && nh > 0 && nkv > 0 && nh % nkv == 0 && q_len > 0 && past_len >= 0 && ldq >= (int64_t)nh * PTTS_HEAD_DIM,
               "op_attention_probs: bad shape");
  PTTS_REQUIRE(kv_len > 0 && kv_len <= capacity && (cross || kv_len == past_len + q_len),
               "op_attention_probs: %d keys (self: past_len + q_len) in a cache of %d positions", kv_len, capacity);
  PTTS_REQUIRE(!rope || (rope_cos && rope_sin), "op_attention_probs: rope needs both tables");
  PTTS_REQUIRE(mask_len >= 0 && (key_mask || mask_len == 0), "op_attention_probs: bad key mask");
  AttnProbeArgs a{};
  a.q = q; a.ldq = ldq; a.q_col0 = 0;
  a.kcache = kcache; a.kv_b_stride = (int64_t)nkv * capacity * PTTS_HEAD_DIM; a.kv_h_stride = (int64_t)capacity * PTTS_HEAD_DIM;
  a.kv_b_div = 1;
  a.key_mask = key_mask; a.mask_len = mask_len; a.mask_ld = mask_len;
  a.B = B; a.nh = nh; a.nkv = nkv; a.q_len = q_len; a.cross = cross ? 1 : 0;
  a.kv_len = kv_len; a.pos0 = past_len; a.kv_cap = kv_len;
  a.rope = rope; a.rope_cos = rope_cos; a.rope_sin = rope_sin; a.scale = 0.125f;
  a.out = out; a.out_q = kv_len; a.out_h = (int64_t)q_len * kv_len; a.out_b = (int64_t)nh * a.out_h;
  return launch_attention_probs(a, dtype, (cudaStream_t)stream);
}

// ---- DAC ----------------------------------------------------------------------------------------
int ptts_dac_blob_bytes(const ptts_dac_config* cfg, int64_t* out_bytes) {
  PTTS_REQUIRE(cfg && out_bytes, "null argument");
  if (int e = validate_dac(*cfg)) return e;
  *out_bytes = make_dac_layout(*cfg).total;
  return PTTS_OK;
}
int ptts_dac_num_tensors(const ptts_dac_config* cfg, int32_t* out) {
  PTTS_REQUIRE(cfg && out, "null argument");
  if (int e = validate_dac(*cfg)) return e;
  *out = (int32_t)make_dac_layout(*cfg).t.size();
  return PTTS_OK;
}
int ptts_dac_pack(const ptts_dac_config* cfg, void* blob, int32_t name_id, const void* src, int32_t src_dtype, int64_t numel, void* stream) {
  PTTS_REQUIRE(cfg && blob && src, "null argument");
  if (int e = validate_dac(*cfg)) return e;
  PTTS_REQUIRE(src_dtype == PTTS_BF16 || src_dtype == PTTS_F32, "dac pack: src dtype must be bf16 or f32");
  const DacLayout L = make_dac_layout(*cfg);
  PTTS_REQUIRE(name_id >= 0 && name_id < (int)L.t.size(), "dac pack: tensor id %d out of range", name_id);
  const DacTensor& t = L.t[name_id];
  PTTS_REQUIRE(numel == t.numel, "dac pack: tensor %d expects %lld elements, got %lld", name_id, (long long)t.numel, (long long)numel);
  char* dst = (char*)blob + t.off;
  if (t.kind == DK_PLAIN) return pack_plain(src, src_dtype, numel, dst, cfg->dtype, (cudaStream_t)stream);
  if (t.off_k >= 0) {
    if (int e = pack_conv_kmajor(src, src_dtype, (char*)blob + t.off_k, t.d0, t.d1, t.k, t.kind == DK_CONVT, (cudaStream_t)stream)) return e;
  }
  return pack_conv(src, src_dtype, dst, cfg->dtype, t.d0, t.d1, t.k, t.kind == DK_CONVT, (cudaStream_t)stream);
}
int ptts_dac_workspace_bytes(const ptts_dac_config* cfg, int32_t B, int32_t T, int64_t* out_bytes) {
  PTTS_REQUIRE(cfg && out_bytes && B > 0 && T > 0, "bad argument");
  if (int e = validate_dac(*cfg)) return e;
  *out_bytes = dac_decode_workspace(*cfg, B, T).bytes();
  return PTTS_OK;
}

int ptts_dac_decode(const ptts_dac_config* cfg, const void* blob, void* workspace, int64_t workspace_bytes, const int64_t* codes,
                    int32_t B, int32_t T, void* audio_out, void* stream) {
  return ptts_dac_decode2(cfg, blob, workspace, workspace_bytes, codes, B, T, nullptr, audio_out, stream);
}

// frame_lengths (device, [B], or NULL): every kernel clamps each value to [0, T], reads no code at or past it and writes zeros
// there (RowLengths in dac.h).
int ptts_dac_decode2(const ptts_dac_config* cfg, const void* blob, void* workspace, int64_t workspace_bytes, const int64_t* codes,
                     int32_t B, int32_t T, const int32_t* frame_lengths, void* audio_out, void* stream) {
  PTTS_REQUIRE(cfg && blob && workspace && codes && audio_out, "null argument");
  if (int e = validate_dac(*cfg)) return e;
  PTTS_REQUIRE(B > 0 && T > 0, "dac decode: empty input B=%d T=%d", B, T);
  PTTS_REQUIRE(workspace_bytes >= dac_decode_workspace(*cfg, B, T).bytes(), "dac decode: workspace too small");
  return dac_decode(*cfg, blob, workspace, codes, B, T, frame_lengths, audio_out, env_flag("PTTS_DAC_TC", true), (cudaStream_t)stream);
}

// Windowed decode: row b decodes codes[b, :, s_b : s_b + n_b] as ptts_dac_decode2 decodes that window alone at frame 0 and keeps the
// samples of window frames [emit_lo[b], emit_hi[b]); each layer computes only the rows those samples depend on (dac.cu).  The
// kernels clamp n_b to [0, T], the emit range to [0, n_b] and s_b to [0, T_codes - n_b].
int ptts_dac_decode3(const ptts_dac_config* cfg, const void* blob, void* workspace, int64_t workspace_bytes, const int64_t* codes,
                     int32_t B, int32_t T_codes, int32_t T, const int32_t* frame_start, const int32_t* frame_lengths,
                     const int32_t* emit_lo, const int32_t* emit_hi, void* audio_out, void* stream) {
  PTTS_REQUIRE(cfg && blob && workspace && codes && audio_out && frame_start && frame_lengths && emit_lo && emit_hi, "null argument");
  if (int e = validate_dac(*cfg)) return e;
  PTTS_REQUIRE(B > 0 && T > 0 && T <= T_codes, "dac decode3: bad shape B=%d T=%d T_codes=%d (0 < T <= T_codes)", B, T, T_codes);
  PTTS_REQUIRE(workspace_bytes >= dac_decode_workspace(*cfg, B, T).bytes(), "dac decode: workspace too small");
  return dac_decode_window(*cfg, blob, workspace, codes, B, T, frame_lengths, DacWindow{frame_start, emit_lo, emit_hi, T_codes}, audio_out,
                           env_flag("PTTS_DAC_TC", true), (cudaStream_t)stream);
}

// ---- DAC encode -----------------------------------------------------------------------------------
int ptts_dac_encoder_blob_bytes(const ptts_dac_config* cfg, int64_t* out_bytes) {
  PTTS_REQUIRE(cfg && out_bytes, "null argument");
  if (int e = validate_dac_encoder(*cfg)) return e;
  *out_bytes = make_dac_enc_layout(*cfg).total;
  return PTTS_OK;
}
int ptts_dac_encoder_num_tensors(const ptts_dac_config* cfg, int32_t* out) {
  PTTS_REQUIRE(cfg && out, "null argument");
  if (int e = validate_dac_encoder(*cfg)) return e;
  *out = (int32_t)make_dac_enc_layout(*cfg).t.size();
  return PTTS_OK;
}
int ptts_dac_encoder_pack(const ptts_dac_config* cfg, void* enc_blob, int32_t name_id, const void* src, int32_t src_dtype, int64_t numel,
                          void* stream) {
  PTTS_REQUIRE(cfg && enc_blob && src, "null argument");
  if (int e = validate_dac_encoder(*cfg)) return e;
  PTTS_REQUIRE(src_dtype == PTTS_BF16 || src_dtype == PTTS_F32, "dac encoder pack: src dtype must be bf16 or f32");
  const DacEncLayout L = make_dac_enc_layout(*cfg);
  PTTS_REQUIRE(name_id >= 0 && name_id < (int)L.t.size(), "dac encoder pack: tensor id %d out of range", name_id);
  const DacEncTensor& t = L.t[name_id];
  PTTS_REQUIRE(numel == t.numel, "dac encoder pack: tensor %d expects %lld elements, got %lld", name_id, (long long)t.numel, (long long)numel);
  cudaStream_t st = (cudaStream_t)stream;
  char* base = (char*)enc_blob;
  switch (t.kind) {
    case EK_PLAIN:
      if (int e = pack_plain(src, src_dtype, numel, base + t.off, cfg->dtype, st)) return e;
      for (int i = 0; t.off_t >= 0 && i < t.tile; i++)
        if (int e = pack_plain(src, src_dtype, numel, base + t.off_t + (int64_t)i * numel * L.es, cfg->dtype, st)) return e;
      return PTTS_OK;
    case EK_CODEBOOK:
      return pack_normalized_codebook(src, src_dtype, (float*)(base + t.off), t.d0, t.d1, cfg->dtype == PTTS_BF16, st);
    case EK_CONV:
      if (t.off_k >= 0)
        if (int e = pack_conv_kmajor(src, src_dtype, base + t.off_k, t.d0, t.d1, t.k, 0, st)) return e;
      return pack_conv(src, src_dtype, base + t.off, cfg->dtype, t.d0, t.d1, t.k, 0, st);
    default:   // EK_SCONV
      if (t.off_k >= 0)
        if (int e = pack_strided_conv(src, src_dtype, base + t.off_k, PTTS_BF16, t.d0, t.d1, t.k / 2, 1, st)) return e;
      return pack_strided_conv(src, src_dtype, base + t.off, cfg->dtype, t.d0, t.d1, t.k / 2, 0, st);
  }
}
int ptts_dac_encode_workspace_bytes(const ptts_dac_config* cfg, int32_t B, int32_t samples, int64_t* out_bytes) {
  PTTS_REQUIRE(cfg && out_bytes && B > 0 && samples > 0, "bad argument");
  if (int e = validate_dac_encoder(*cfg)) return e;
  *out_bytes = dac_encode_workspace(*cfg, B, samples).bytes();
  return PTTS_OK;
}

int ptts_dac_encode(const ptts_dac_config* cfg, const void* dec_blob, const void* enc_blob, void* workspace, int64_t workspace_bytes,
                    const void* audio, int32_t B, int32_t samples, int32_t n_q, int64_t* codes_out, void* latents_out, void* stream) {
  return ptts_dac_encode2(cfg, dec_blob, enc_blob, workspace, workspace_bytes, audio, B, samples, nullptr, n_q, codes_out, latents_out,
                          stream);
}

// sample_lengths (device, [B], or NULL): every kernel clamps each value to [1, samples], reads no sample at or past it, and the
// frames past the row's ceil(n_b / hop) hold codebook_size and zero latents (RowLengths in dac.h).
int ptts_dac_encode2(const ptts_dac_config* cfg, const void* dec_blob, const void* enc_blob, void* workspace, int64_t workspace_bytes,
                     const void* audio, int32_t B, int32_t samples, const int32_t* sample_lengths, int32_t n_q, int64_t* codes_out,
                     void* latents_out, void* stream) {
  PTTS_REQUIRE(cfg && dec_blob && enc_blob && workspace && audio && codes_out, "null argument");
  if (int e = validate_dac_encoder(*cfg)) return e;
  PTTS_REQUIRE(B > 0 && samples > 0, "dac encode: empty input B=%d samples=%d", B, samples);
  PTTS_REQUIRE(n_q >= 1 && n_q <= cfg->n_codebooks, "dac encode: n_q %d outside 1..%d", n_q, cfg->n_codebooks);
  PTTS_REQUIRE(workspace_bytes >= dac_encode_workspace(*cfg, B, samples).bytes(), "dac encode: workspace too small");
  return dac_encode(*cfg, dec_blob, enc_blob, workspace, audio, B, samples, sample_lengths, n_q, codes_out, latents_out,
                    env_flag("PTTS_DAC_TC", true), (cudaStream_t)stream);
}

// One codec conv launch (test hook).  The geometry comes from the dac.h constructors and the weights go through the packs the
// blobs use, so that both are under test with the kernel.
int ptts_op_dac_conv(int32_t dtype, int32_t kernel, int32_t kind, int32_t B, int32_t Cin, int32_t Cout, int32_t T, int32_t taps,
                     int32_t dil_or_stride, int32_t samples, const void* weight, const void* bias, const void* alpha,
                     const void* alpha_next, const void* x, const void* res, void* out_raw, void* out_act, int32_t tanh_out,
                     const int32_t* frame_lengths, int32_t frames, void* scratch, void* stream) {
  PTTS_REQUIRE(weight && bias && x && scratch && (out_raw || out_act), "null argument");
  PTTS_REQUIRE(dtype == PTTS_BF16 || dtype == PTTS_F32, "op_dac_conv: dtype must be bf16 or f32");
  PTTS_REQUIRE(kernel >= 0 && kernel <= 3, "op_dac_conv: kernel is 0 (conv_kernel), 1 (conv_tc_kernel), 2 (final conv) or 3 (input conv)");
  PTTS_REQUIRE(kind >= 0 && kind <= 2, "op_dac_conv: kind is 0 (conv_same), 1 (conv_up) or 2 (conv_super_rows)");
  PTTS_REQUIRE(B > 0 && Cin > 0 && Cout > 0 && T > 0 && taps > 0 && dil_or_stride > 0, "op_dac_conv: bad shape");
  PTTS_REQUIRE(kernel == 0 || dtype == PTTS_BF16, "op_dac_conv: kernel %d is bf16 only", kernel);
  PTTS_REQUIRE(kind == 0 || dil_or_stride % 2 == 0, "op_dac_conv: stride %d must be even", dil_or_stride);
  PTTS_REQUIRE(kind != 2 || T % dil_or_stride == 0, "op_dac_conv: conv_super_rows needs T %% s == 0");
  PTTS_REQUIRE(frame_lengths == nullptr || frames > 0, "op_dac_conv: frame_lengths needs frames > 0");
  const int s = dil_or_stride;
  ConvArgs a = kind == 0 ? conv_same(Cin, Cout, T, taps, dil_or_stride) : kind == 1 ? conv_up(Cin, Cout, T, s) : conv_super_rows(Cin, Cout, T, s);
  a.x = x; a.bias = bias; a.res = res;
  const int k_src = kind == 0 ? taps : 2 * s;   // taps of the PyTorch weight
  cudaStream_t st = (cudaStream_t)stream;
  auto ragged = [&](const ConvArgs& c) {
    if (frame_lengths == nullptr) return RowLengths{};
    return RowLengths{frame_lengths, frames, c.Tin / frames, c.Tout / frames};
  };
  PTTS_REQUIRE(frame_lengths == nullptr || (a.Tin % frames == 0 && a.Tout % frames == 0), "op_dac_conv: %d / %d rows are not whole frames of %d",
               a.Tin, a.Tout, frames);
  switch (kernel) {
    case 0: {   // conv_kernel, snake_alpha on the input; alpha of a strided conv tiled s times over the super-row channels
      PTTS_REQUIRE(!alpha_next && !out_act && out_raw, "op_dac_conv: conv_kernel writes out_raw only");
      PTTS_REQUIRE(samples == 0 || (kind == 0 && samples > 0 && samples <= T), "op_dac_conv: samples is for conv_same only, 1..T");
      if (samples > 0) a.Tin = samples;   // the encoder's input conv: rows past `samples` read zeros
      const int es = dtype_size(dtype);
      if (kind == 2) {
        if (int e = pack_strided_conv(weight, dtype, scratch, dtype, Cout, Cin, s, 0, st)) return e;
      } else if (int e = pack_conv(weight, dtype, scratch, dtype, kind == 1 ? Cin : Cout, kind == 1 ? Cout : Cin, k_src, kind == 1, st)) {
        return e;
      }
      a.w = scratch;
      a.alpha = alpha;
      if (kind == 2 && alpha != nullptr) {
        char* tiled = (char*)scratch + align_up((int64_t)3 * s * Cin * Cout * es, 256);
        for (int i = 0; i < s; i++)
          if (int e = pack_plain(alpha, dtype, Cin, tiled + (int64_t)i * Cin * es, dtype, st)) return e;
        a.alpha = tiled;
      }
      a.out = out_raw; a.tanh_out = tanh_out ? 1 : 0;
      return launch_conv(a, dtype, B, st, ragged(a));
    }
    case 1: {   // conv_tc_kernel: snake_{alpha_next} of the output
      PTTS_REQUIRE(conv_tc_supported(a.Cin, a.Cout), "op_dac_conv: conv_tc_kernel does not take Cin %d, Cout %d", a.Cin, a.Cout);
      PTTS_REQUIRE(!alpha && !tanh_out && samples == 0, "op_dac_conv: conv_tc_kernel has no input snake, tanh or samples");
      PTTS_REQUIRE(!out_act == !alpha_next, "op_dac_conv: out_act and alpha_next go together");
      if (kind == 2) {
        if (int e = pack_strided_conv(weight, dtype, scratch, PTTS_BF16, Cout, Cin, s, 1, st)) return e;
      } else if (int e = pack_conv_kmajor(weight, dtype, scratch, kind == 1 ? Cin : Cout, kind == 1 ? Cout : Cin, k_src, kind == 1, st)) {
        return e;
      }
      return launch_conv_tc(a, scratch, a.n_taps * a.n_phase, alpha_next, out_raw, out_act, B, st, ragged(a));
    }
    case 2: {   // final_conv_tanh_kernel over an already snake'd input
      PTTS_REQUIRE(kind == 0 && Cout == 1 && taps == 7 && dil_or_stride == 1 && final_conv_supported(Cin),
                   "op_dac_conv: the final conv is conv_same(C, 1, T, 7, 1) with final_conv_supported(C), got Cin %d Cout %d taps %d", Cin, Cout, taps);
      PTTS_REQUIRE(!alpha && !alpha_next && !res && !out_act && out_raw && tanh_out && samples == 0, "op_dac_conv: the final conv writes tanh to out_raw only");
      if (int e = pack_conv(weight, dtype, scratch, dtype, Cout, Cin, 7, 0, st)) return e;
      return launch_final_conv_tanh(x, scratch, bias, out_raw, Cin, T, B, frame_lengths, frames, st);
    }
    default: {  // enc_input_conv_kernel: T rows from `samples` waveform samples, raw and snake_{alpha_next}
      PTTS_REQUIRE(kind == 0 && Cin == 1 && taps == 7 && dil_or_stride == 1 && samples > 0 && samples <= T,
                   "op_dac_conv: the input conv is conv_same(1, C, T, 7, 1) over 1..T samples");
      PTTS_REQUIRE(!alpha && !res && !tanh_out && !frame_lengths && alpha_next && out_raw && out_act, "op_dac_conv: the input conv writes raw and snake_{alpha_next}");
      if (int e = pack_conv(weight, dtype, scratch, dtype, Cout, 1, 7, 0, st)) return e;
      return launch_enc_input_conv(x, scratch, bias, alpha_next, out_raw, out_act, Cout, samples, T, B, nullptr, 0, st);
    }
  }
}

}  // extern "C"
