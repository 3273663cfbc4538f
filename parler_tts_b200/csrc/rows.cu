// rows.cu -- moving batch rows between sessions (continuous batching): the per-row state of row_regions (layout.h) copied from
// the rows of one session into slots of another, and the control-block rewrite of ptts_generate_set_slots2.
#include "common.cuh"
#include "kernels.h"

namespace ptts {

// grid (pair, region, i): CTA (p, r, i) copies the blocks (i, *, *) of region r for row pair p.  K/V rows keep their swizzle:
// kv_swz depends on the position only, and a block is a row's positions [0, kv_len) of one head.
__global__ void __launch_bounds__(256) import_rows_kernel(RowImportArgs a) {
  const int p = blockIdx.x, r = blockIdx.y, i = blockIdx.z;
  const RowRegion& s = a.src[r];
  const RowRegion& d = a.dst[r];
  if (i >= s.n[0]) return;
  int64_t bytes = s.bytes < d.bytes ? s.bytes : d.bytes;
  const int src_len = a.src_ctrl->cur_len, dst_len = a.dst_ctrl->cur_len;
  if (s.kind == ROW_HISTORY) bytes = min(bytes, (int64_t)src_len * 8);
  const char* sb = a.src_ws + s.off + i * s.stride[0] + a.src_row[p] * s.row_stride + (src_len & 1) * s.parity;
  char* db = a.dst_ws + d.off + i * d.stride[0] + a.dst_row[p] * d.row_stride + (dst_len & 1) * d.parity;
  if (s.kind == ROW_FIRST_UNF) {
    if (threadIdx.x == 0) *(int*)db = *(const int*)sb + (a.dst_row[p] - a.src_row[p]) * a.K;
    return;
  }
  for (int j = 0; j < s.n[1]; j++)
    for (int l = 0; l < s.n[2]; l++) {
      const char* src = sb + j * s.stride[1] + l * s.stride[2];
      char* dst = db + j * d.stride[1] + l * d.stride[2];
      if ((((uintptr_t)src | (uintptr_t)dst | (uintptr_t)bytes) & 15) == 0) {
        for (int64_t o = threadIdx.x; o < bytes / 16; o += blockDim.x) ((int4*)dst)[o] = __ldg((const int4*)src + o);
      } else {   // every region is whole 4-byte words (a mask row, a codebook's ids)
        for (int64_t o = threadIdx.x; o < bytes / 4; o += blockDim.x) ((int*)dst)[o] = __ldg((const int*)src + o);
      }
    }
}

int launch_import_rows(const RowImportArgs& a, int n_pairs, cudaStream_t st) {
  int z = 1;
  for (int r = 0; r < a.n_regions; r++) z = a.src[r].n[0] > z ? a.src[r].n[0] : z;
  import_rows_kernel<<<dim3(n_pairs, a.n_regions, z), 256, 0, st>>>(a);
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

// the rows come by value (the host's arrays need no staging copy and no stream sync); the first launch also writes the control block
struct SlotRows {
  int* shift; int* key; int* max_len;   // the workspace's row_shift, row_key and row_max_len
  int b0, n;
  int v_shift[kMaxSlotRows], v_key[kMaxSlotRows], v_max_len[kMaxSlotRows];
};
__global__ void set_slots_kernel(Ctrl* ctrl, int cur_len, SlotRows r) {
  for (int i = threadIdx.x; i < r.n; i += blockDim.x) {
    r.shift[r.b0 + i] = r.v_shift[i]; r.key[r.b0 + i] = r.v_key[i]; r.max_len[r.b0 + i] = r.v_max_len[i];
  }
  if (r.b0 == 0 && threadIdx.x == 0) {
    ctrl->cur_len = cur_len;
    ctrl->active = 1;
    ctrl->n_unfinished = 0;
    ctrl->done_blocks = 0;
  }
}

int launch_set_slots(Ctrl* ctrl, int cur_len, int* shift, int* key, int* max_len, const int* row_shift, const int* row_key,
                     const int* row_max_len, int B, cudaStream_t st) {
  for (int b0 = 0; b0 < B; b0 += kMaxSlotRows) {
    SlotRows r{};
    r.shift = shift; r.key = key; r.max_len = max_len; r.b0 = b0; r.n = B - b0 < kMaxSlotRows ? B - b0 : kMaxSlotRows;
    for (int i = 0; i < r.n; i++) { r.v_shift[i] = row_shift[b0 + i]; r.v_key[i] = row_key[b0 + i]; r.v_max_len[i] = row_max_len[b0 + i]; }
    set_slots_kernel<<<1, 256, 0, st>>>(ctrl, cur_len, r);
    PTTS_LAUNCH_CHECK();
  }
  return PTTS_OK;
}

}  // namespace ptts
