// layout.h -- byte layout of the packed decoder weight blob and of the generation workspace.
//
// HBM layout (DESIGN.md "Data layout"):
//   blob      : [embed tables K x (V+1) x H][pos table][L x layer][final LN][lm heads (K*V) x H]
//               GEMM matrices are stored in mma.m16n8k16 B-fragment order (bf16) so a warp's 512 B
//               load is one fully coalesced request and needs no shared-memory staging.
//   workspace : control block, token history, activations, cross K/V [L][(B/takes)*S][2*nckv*64],
//               self K/V cache [L][2][B][nkv][Tmax][64].
#pragma once
#include "common.cuh"

namespace ptts {

struct DecoderLayout {
  int es;  // element size of model dtype
  int H, F, V, K, L, nh, nkv, nckv, qkv_rows, ckv_rows;
  int64_t embed, pos, layer0, layer_stride;
  // offsets inside one layer
  int64_t ln1_w, ln1_b, wqkv, wo, ln2_w, ln2_b, wqc, wkvc, woc, ln3_w, ln3_b, fc1, fc2;
  int64_t c_qkv, c_qc, c_fc1;   // folded-LayerNorm vectors (c1 | c2), f32, per layer (ln_stats.cuh)
  int64_t final_ln_w, final_ln_b, heads, rope_cos, rope_sin, c_heads;
  // cluster step kernel (step2.cu): a second copy of the six per-layer matrices, cut into one contiguous slice per
  // (phase, cluster, rank): the n-tiles the cluster owns x the K range the rank reduces.  cl_NC == 0: shape not covered.
  int cl_C, cl_NC;          // CTAs per cluster (2), clusters (4 per head)
  int64_t rm[7];            // per layer (bf16 only): ROW-MAJOR copies of wqkv, wo, wqc, wkvc, woc, fc1, fc2 for the wgmma prefill
                            // GEMM (gemm_tc.cu: TMA-tiled K-major operands); indexed by DecoderMatrixId
  int64_t cp[6];            // per layer: offset of phase p's slices (A qkv | B o | C q_cross | D o_cross | E fc1 | F fc2)
  int64_t cp_slice[6];      // bytes of one (cluster, rank) slice of phase p
  int64_t total;
};

// Shapes the cluster step kernel covers: bf16, MHA for self- and cross-attention, four clusters of 2 CTAs per head (at most 18 heads;
// whether the device holds the grid co-resident is asked at session set-up, step2.cu cluster_step_available: a 132-SM H100 holds
// 66 clusters of 2, i.e. up to 16 heads), K a whole number of 8-tile groups (step.cu's 8-way K split), H / (4 heads) = 16 out-proj features per cluster, at
// most 4 fc1 n-tiles per rank, and the shared-memory plan of step2.cu (sized for H <= 1024, F <= 4096).
static inline bool cluster_shape_ok(const ptts_decoder_config& c) {
  const int H = c.hidden_size, nh = c.num_heads, F = c.ffn_dim;
  return c.dtype == PTTS_BF16 && c.num_kv_heads == nh && c.num_cross_kv_heads == nh && nh * 8 <= 144 && H == nh * PTTS_HEAD_DIM &&
         H % 256 == 0 && F % 256 == 0 && F % (nh * 64) == 0 && (F / (nh * 64) == 1 || F / (nh * 64) == 2 || F / (nh * 64) == 4) && H <= 1024 && F <= 4096 && c.num_codebooks <= 16 &&
         (c.vocab_size * c.num_codebooks) % 32 == 0;
}

static inline int dtype_size(int dt) { return dt == PTTS_BF16 ? 2 : 4; }

// Cluster step kernel (step2.cu): how phase ph of a layer (A qkv | B o | C q_cross | D o_cross | E fc1 | F fc2) cuts its matrix
// into slices.  A slice is nt n-tiles (a head's q|k|v = 192 features, a cluster's 16 out-proj features, a head's q_cross, ...,
// F / (4 nh) fc1 features) x the kt k32 tiles of one rank; the head phases keep one slice set per head, the others one per cluster.
struct ClusterPhase {
  int64_t mat;     // offset of the fragment-order matrix inside the layer
  int nt, owners;  // n-tiles per slice; slice owners (heads or clusters), each with cl_C slices
  int kt, kt_src;  // k32 tiles per rank; of the whole matrix
};
static inline ClusterPhase cluster_phase(const DecoderLayout& l, int ph) {
  const int64_t mat[6] = {l.wqkv, l.wo, l.wqc, l.woc, l.fc1, l.fc2};
  const int nt[6] = {24, 2, 8, 2, l.F / (4 * l.nh) / 8, 2};
  const int owners[6] = {l.nh, 4 * l.nh, l.nh, 4 * l.nh, 4 * l.nh, 4 * l.nh};
  const int K = (ph == 5) ? l.F : l.H;
  return {mat[ph], nt[ph], owners[ph], K / l.cl_C / 32, K / 32};
}

static inline DecoderLayout make_layout(const ptts_decoder_config& c) {
  DecoderLayout l{};
  l.es = dtype_size(c.dtype);
  l.H = c.hidden_size; l.F = c.ffn_dim; l.V = c.vocab_size; l.K = c.num_codebooks; l.L = c.num_layers;
  l.nh = c.num_heads; l.nkv = c.num_kv_heads; l.nckv = c.num_cross_kv_heads;
  l.qkv_rows = (l.nh + 2 * l.nkv) * PTTS_HEAD_DIM;
  l.ckv_rows = 2 * l.nckv * PTTS_HEAD_DIM;
  int64_t o = 0;
  auto take = [&](int64_t bytes) { int64_t r = o; o = align_up(o + bytes, 256); return r; };
  l.embed = take((int64_t)l.K * (l.V + 1) * l.H * l.es);
  l.pos = take(c.rope ? 0 : (int64_t)c.max_positions * l.H * l.es);
  l.layer0 = o;
  int64_t base = o;
  l.ln1_w = take(l.H * 4) - base; l.ln1_b = take(l.H * 4) - base;
  l.wqkv = take((int64_t)l.qkv_rows * l.H * l.es) - base;
  l.wo = take((int64_t)l.H * l.H * l.es) - base;
  l.ln2_w = take(l.H * 4) - base; l.ln2_b = take(l.H * 4) - base;
  l.wqc = take((int64_t)l.H * l.H * l.es) - base;
  l.wkvc = take((int64_t)l.ckv_rows * l.H * l.es) - base;
  l.woc = take((int64_t)l.H * l.H * l.es) - base;
  l.ln3_w = take(l.H * 4) - base; l.ln3_b = take(l.H * 4) - base;
  l.fc1 = take((int64_t)l.F * l.H * l.es) - base;
  l.fc2 = take((int64_t)l.H * l.F * l.es) - base;
  l.c_qkv = take((int64_t)2 * l.qkv_rows * 4) - base;
  l.c_qc = take((int64_t)2 * l.H * 4) - base;
  l.c_fc1 = take((int64_t)2 * l.F * 4) - base;
  for (int i = 0; i < 7; i++) l.rm[i] = 0;
  if (c.dtype == PTTS_BF16) {
    const int64_t sz[7] = {(int64_t)l.qkv_rows * l.H, (int64_t)l.H * l.H, (int64_t)l.H * l.H, (int64_t)l.ckv_rows * l.H, (int64_t)l.H * l.H,
                           (int64_t)l.F * l.H, (int64_t)l.H * l.F};
    for (int i = 0; i < 7; i++) l.rm[i] = take(sz[i] * 2) - base;
  }
  l.cl_C = l.cl_NC = 0;
  for (int i = 0; i < 6; i++) l.cp[i] = l.cp_slice[i] = 0;
  if (cluster_shape_ok(c)) {
    l.cl_C = 2; l.cl_NC = 4 * l.nh;
    for (int i = 0; i < 6; i++) {
      const ClusterPhase cp = cluster_phase(l, i);
      l.cp_slice[i] = (int64_t)cp.nt * cp.kt * 512;
      l.cp[i] = take(l.cp_slice[i] * cp.owners * l.cl_C) - base;
    }
  }
  l.layer_stride = o - base;
  o = base + l.layer_stride * l.L;
  l.final_ln_w = take(l.H * 4); l.final_ln_b = take(l.H * 4);
  l.heads = take((int64_t)l.K * l.V * l.H * l.es);
  l.rope_cos = take(c.rope ? (int64_t)c.max_positions * PTTS_HEAD_DIM * l.es : 0);
  l.rope_sin = take(c.rope ? (int64_t)c.max_positions * PTTS_HEAD_DIM * l.es : 0);
  l.c_heads = take((int64_t)2 * l.K * l.V * 4);
  l.total = o;
  return l;
}

static inline int validate_config(const ptts_decoder_config& c) {
  PTTS_REQUIRE(c.dtype == PTTS_BF16 || c.dtype == PTTS_F32, "dtype must be bf16(0) or f32(1), got %d", c.dtype);
  PTTS_REQUIRE(c.hidden_size > 0 && c.num_heads > 0 && c.hidden_size == c.num_heads * PTTS_HEAD_DIM,
               "hidden_size (%d) must equal num_heads (%d) * %d", c.hidden_size, c.num_heads, PTTS_HEAD_DIM);
  PTTS_REQUIRE(c.num_kv_heads > 0 && c.num_heads % c.num_kv_heads == 0, "num_heads %% num_kv_heads != 0");
  PTTS_REQUIRE(c.num_cross_kv_heads > 0 && c.num_heads % c.num_cross_kv_heads == 0, "num_heads %% num_cross_kv_heads != 0");
  PTTS_REQUIRE(c.hidden_size % 32 == 0 && c.ffn_dim % 32 == 0, "hidden_size and ffn_dim must be multiples of 32");
  PTTS_REQUIRE(c.ffn_dim % c.hidden_size == 0, "ffn_dim must be a multiple of hidden_size");
  PTTS_REQUIRE(c.vocab_size % 8 == 0, "vocab_size must be a multiple of 8, got %d", c.vocab_size);
  PTTS_REQUIRE(c.hidden_size <= 2048, "hidden_size > 2048 not supported by the activation tile");
  PTTS_REQUIRE(c.num_codebooks >= 1 && c.num_codebooks <= 32, "num_codebooks out of range");
  PTTS_REQUIRE(c.num_layers >= 1 && c.activation >= 0 && c.activation <= 3, "bad num_layers/activation");
  return PTTS_OK;
}

// The decoder's GEMM matrices: the seven of each layer (fused where the reference has several projections) and the lm heads.
enum DecoderMatrixId { MAT_QKV, MAT_O, MAT_Q_CROSS, MAT_KV_CROSS, MAT_O_CROSS, MAT_FC1, MAT_FC2, MAT_HEADS, MAT_COUNT };
struct DecoderMatrix {
  int64_t w;           // blob offset of the fragment-order weights
  int N, K;            // rows = output features, columns
  int64_t ln_w, ln_b;  // blob offsets of the fp32 gamma / beta of the LayerNorm in front; -1: none
  int64_t c;           // blob offset of the folded LayerNorm vectors c1 | c2 (fp32, N each; bf16 only, ptts_decoder_finalize); -1: none
  int64_t rm;          // blob offset of the row-major copy the wgmma prefill GEMM reads; -1: none (f32, or the lm heads)
};
// Matrix m of `layer` (ignored for the lm heads).
static inline DecoderMatrix decoder_matrix(const DecoderLayout& l, int m, int layer) {
  const int64_t lb = l.layer0 + l.layer_stride * layer;
  const int64_t rm = l.es == 2 && m != MAT_HEADS ? lb + l.rm[m] : -1;
  switch (m) {
    case MAT_QKV: return {lb + l.wqkv, l.qkv_rows, l.H, lb + l.ln1_w, lb + l.ln1_b, lb + l.c_qkv, rm};
    case MAT_O: return {lb + l.wo, l.H, l.H, -1, -1, -1, rm};
    case MAT_Q_CROSS: return {lb + l.wqc, l.H, l.H, lb + l.ln2_w, lb + l.ln2_b, lb + l.c_qc, rm};
    case MAT_KV_CROSS: return {lb + l.wkvc, l.ckv_rows, l.H, -1, -1, -1, rm};
    case MAT_O_CROSS: return {lb + l.woc, l.H, l.H, -1, -1, -1, rm};
    case MAT_FC1: return {lb + l.fc1, l.F, l.H, lb + l.ln3_w, lb + l.ln3_b, lb + l.c_fc1, rm};
    case MAT_FC2: return {lb + l.fc2, l.H, l.F, -1, -1, -1, rm};
    default: return {l.heads, l.K * l.V, l.H, l.final_ln_w, l.final_ln_b, l.c_heads, -1};
  }
}

// An ABI tensor id's place in the matrix table: the fused matrix and the tensor's first row in it.
struct MatSlot {
  DecoderMatrix m;
  int row_off;
};
// Resolve (tensor_id, index) -> fused matrix slot (index: the layer, or the lm head's codebook).  Returns false for non-matrix tensors.
static inline bool matrix_slot(const DecoderLayout& l, int tensor_id, int index, MatSlot* s) {
  const int D = PTTS_HEAD_DIM;
  auto slot = [&](int m, int row_off) { *s = {decoder_matrix(l, m, index), row_off}; return true; };
  switch (tensor_id) {
    case PTTS_T_SELF_Q: return slot(MAT_QKV, 0);
    case PTTS_T_SELF_K: return slot(MAT_QKV, l.nh * D);
    case PTTS_T_SELF_V: return slot(MAT_QKV, (l.nh + l.nkv) * D);
    case PTTS_T_SELF_O: return slot(MAT_O, 0);
    case PTTS_T_CROSS_Q: return slot(MAT_Q_CROSS, 0);
    case PTTS_T_CROSS_K: return slot(MAT_KV_CROSS, 0);
    case PTTS_T_CROSS_V: return slot(MAT_KV_CROSS, l.nckv * D);
    case PTTS_T_CROSS_O: return slot(MAT_O_CROSS, 0);
    case PTTS_T_FC1: return slot(MAT_FC1, 0);
    case PTTS_T_FC2: return slot(MAT_FC2, 0);
    case PTTS_T_LM_HEAD: return slot(MAT_HEADS, index * l.V);
    default: return false;
  }
}

// ---- workspace ----------------------------------------------------------------------------------
struct WorkspaceLayout {
  int B, P, S, Tmax, Mmax, BK;
  int takes;                       // consecutive rows per description: cross K/V and enc_mask hold B / takes descriptions
  int max_input;                   // largest decoder input (BOS column + code prefix) a generate() call may continue from
  int64_t ctrl, progress, gen, raw_ids, cur_ids, eos_seen, unfinished, first_unf, prompt_mask, enc_mask;
  int64_t prefix_cells;            // [BK][K-1] int64: delay-pattern cells just past the input (max_input > 1 only; -1 = none)
  int64_t row_shift;               // [B] int32: per-row offsets of a ragged continuation (max_input > 1 only; -1 = none)
  int64_t x, qkv, attn, qc, hbuf, hidden, logits, scores, cross_tmp, cross_kv, self_kv;
  int64_t img_x, img_attn, img_h;  // fused step kernel: activations as tile images [chunk][32][H + 8] (step.cu stage_tile)
  int64_t cl_x, cl_attn, cl_h;     // cluster step kernel: K-sliced images [2][32][H/2 + 8], fc2's in quarters [4][32][F/4 + 8] (step2.cu)
  int64_t row_stats;               // [max(B*(P+max_input), B*S)][2] f32: LayerNorm row statistics of the wgmma prefill GEMMs
  int64_t cross_layer_stride, self_layer_stride;  // bytes
  int64_t raw_ld;                                  // raw_ids leading dimension (elements)
  int64_t total;
};

// max_input = 1: the BOS column only; the layout is then the same as before continuation existed (prefix_cells takes no bytes).
// takes (divides B): rows b .. b + takes - 1 of each group are takes of one description and read its cross K/V; takes = 1 is the
// layout of one description per row.  Only the cross K/V (and its re-layout buffer) and enc_mask depend on it.
static inline WorkspaceLayout make_workspace(const ptts_decoder_config& c, int B, int P, int S, int Tmax, int max_input = 1, int takes = 1) {
  DecoderLayout l = make_layout(c);
  WorkspaceLayout w{};
  w.B = B; w.P = P; w.S = S; w.Tmax = Tmax; w.BK = B * c.num_codebooks;
  w.takes = takes;
  w.max_input = max_input;
  w.Mmax = B * (P + max_input);
  int64_t o = 0;
  auto take = [&](int64_t bytes) { int64_t r = o; o = align_up(o + bytes, 256); return r; };
  w.ctrl = take(sizeof(Ctrl));
  w.progress = take(1024 * 4);
  w.gen = take(sizeof(ptts_gen_params));
  w.raw_ld = Tmax - P + 1;  // >= max_length
  w.raw_ids = take((int64_t)w.BK * w.raw_ld * 8);
  w.cur_ids = take((int64_t)w.BK * 4);
  w.eos_seen = take((int64_t)w.BK * 4);
  w.unfinished = take((int64_t)w.BK * 4);
  w.first_unf = take((int64_t)2 * B * 4);
  w.prompt_mask = take((int64_t)B * (P > 0 ? P : 1) * 4);
  w.enc_mask = take((int64_t)(B / takes) * S * 4);
  w.prefix_cells = -1;
  if (max_input > 1 && c.num_codebooks > 1) w.prefix_cells = take((int64_t)w.BK * (c.num_codebooks - 1) * 8);
  w.row_shift = max_input > 1 ? take((int64_t)B * 4) : -1;
  const int64_t rows_enc = (int64_t)B * S, rows_cross = (int64_t)(B / takes) * S;
  w.x = take((int64_t)w.Mmax * l.H * l.es);
  w.qkv = take((int64_t)w.Mmax * l.qkv_rows * l.es);
  w.attn = take((int64_t)w.Mmax * l.H * l.es);
  w.qc = take((int64_t)w.Mmax * l.H * l.es);
  w.hbuf = take((int64_t)w.Mmax * l.F * l.es);
  w.hidden = take((int64_t)B * l.H * l.es);
  w.img_x = take((int64_t)32 * (l.H + 8) * 2);
  w.img_attn = take((int64_t)32 * (l.H + 8) * 2);
  w.img_h = take((int64_t)((l.F + l.H - 1) / l.H) * 32 * (l.H + 8) * 2);
  w.row_stats = take((int64_t)(w.Mmax > rows_enc ? w.Mmax : rows_enc) * 2 * 4);
  w.cl_x = take((int64_t)2 * 32 * (l.H / 2 + 8) * 2);
  w.cl_attn = take((int64_t)2 * 32 * (l.H / 2 + 8) * 2);
  w.cl_h = take((int64_t)4 * 32 * (l.F / 4 + 8) * 2);
  w.logits = take((int64_t)w.BK * l.V * 4);
  w.scores = take((int64_t)w.BK * l.V * 4);
  w.cross_layer_stride = align_up(rows_cross * l.ckv_rows * l.es, 256);
  w.cross_tmp = take(w.cross_layer_stride);   // GEMM output of one layer before the item-major re-layout
  w.cross_kv = take(w.cross_layer_stride * l.L);
  w.self_layer_stride = align_up((int64_t)2 * B * l.nkv * Tmax * PTTS_HEAD_DIM * l.es, 256);
  w.self_kv = take(w.self_layer_stride * l.L);
  w.total = o;
  return w;
}

}  // namespace ptts
