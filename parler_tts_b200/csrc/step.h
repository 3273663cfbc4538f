// step.h -- parameters of the fused decode-step kernels (step.cu, step2.cu).
#pragma once
#include "common.cuh"
#include "kernels.h"
#include "layout.h"

namespace ptts {

struct StepParams {
  // shapes
  int B, H, F, V, K, L, nh, nkv, nckv, S, P, Tmax, rope, act, qkv_rows, ckv_rows;
  int takes;               // consecutive rows that share one description's cross K/V and encoder mask (B / takes of each)
  float eps, scale;
  // packed weights: blob offsets from the session's layout (the cluster kernel's weight slices: lay.cp, lay.cp_slice)
  const char* blob;
  DecoderLayout lay;
  // workspace
  bf16 *x, *qkv, *attn, *qc, *hbuf;  // x / attn / hbuf are tile images (row pitch H + 8; hbuf: F/H images), qkv / qc plain rows
  float* logits;
  char* cross_kv; int64_t cross_layer_stride;
  char* self_kv; int64_t self_layer_stride;
  const int* prompt_mask;  // nullable
  const int* enc_mask;     // nullable
  SampleArgs sa;
  unsigned* bar;           // [2] device-wide barrier counters (Ctrl::bar)
  // schedule (plan_decode_step)
  int nt_qkv, nt_h, nt_fc1, nt_heads;
  int nbuf;                // activation-tile buffers (2 = double-buffered K chunks)
  int64_t tile_region_bytes;   // scratch after the header: [activation tiles | weight buffer], aliased by attention
  int64_t wbuf_offset;         // weight buffer offset inside the scratch region
  int do_sample_phase;     // 1: logits -> token inside the kernel (ptts_decode_steps); 0: stop at the logits
  int sample_items;        // ceil(V / 256): logits per thread of the one-CTA-per-row sampler
  int* progress;           // debug: last phase each CTA arrived at (printed on a barrier timeout)
  int n_steps;             // cluster kernel: tokens one launch may run (stops early when every row is finished); 0 / 1 = one
  long long* prof;         // optional [(8L+3)][8] clock64 timestamps written by CTA 0 (debug / profiles)
  // ---- cluster step kernel (step2.cu) ----
  bf16 *cl_x, *cl_attn, *cl_h;  // K-sliced activation images [slices][32][slice width + 8]: x, attn 2 slices of H/2; h 4 of F/4
};

// Plans step.cu's launch on a grid of `grid` CTAs for the shape in p: n-tiles per task, tile buffers, the shared-memory region
// and the sampler width.  Returns nullptr, or why step.cu does not take the shape.
const char* plan_decode_step(StepParams& p, int grid);
int launch_decode_step(const StepParams& p, int grid, cudaStream_t st);
// cluster step kernel (step2.cu)
bool cluster_step_available(const StepParams& p);
int launch_decode_step_cluster(const StepParams& p, cudaStream_t st);
// the (phase, cluster or head, rank) weight slices of one layer (blob bytes at `layer`), cut from its fragment-order matrices
int cluster_pack_layer(const DecoderLayout& L, char* layer, cudaStream_t st);

}  // namespace ptts
