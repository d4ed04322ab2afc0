// wvn-b200: internal interface of segment_kernels.cu.
#pragma once

#include <cuda_runtime.h>

namespace wvn {

struct SegmentArgs {
  int batch = 0;
  int h = 0, w = 0;            // segmentation map size
  int smax = 0;                // segment ids are in [0, smax); others (e.g. -1) are ignored
  int grid_h = 0, grid_w = 0;  // token grid the dense features would be upsampled from
  int dim = 0;                 // feature channels
  float scale_y = 0.f, scale_x = 0.f;  // (grid-1)/(out-1): align_corners=True upsampling to (h, h)
};

// stats: [B, smax, 3] u64 = (count, sum of col, sum of row); wseg: [B, smax, grid_h*grid_w] f32 or null;
// adj: [B, smax, ceil(smax/32)] u32 bitset (row = right/bottom id, bit = left/top id) or null.
int segment_accumulate(const long long* seg, const SegmentArgs& a, unsigned long long* stats, float* wseg,
                       unsigned int* adj, cudaStream_t stream);
// feat: [B, smax, dim] f32 or null; centers: [B, smax, 2] f32 (x=col, y=row) or null.
int segment_pool(const float* wseg, const float* tokens, const unsigned long long* stats, float* feat, float* centers,
                 const SegmentArgs& a, cudaStream_t stream);
// edges: [B, max_edges, 2] i64 (le, ri), sorted by (ri, le); n_edges: [B] i32.
int adjacency_emit(const unsigned int* adj, long long* edges, int* n_edges, int batch, int smax, int max_edges,
                   cudaStream_t stream);
// In-place relabel of each frame's labels to 0..S-1 (ascending label order); scratch: [B, num_labels] i32
// (becomes the remap table), counts: [B] i32 = S per frame.
int relabel_compact(long long* seg, int* scratch, int* counts, int batch, long long pix_per_frame, int num_labels,
                    cudaStream_t stream);

// Per-segment mean of a supervision mask (NaN = unlabelled), nodes.py:400-440.  mask: [B, C, h, w] f32;
// y: [B, smax] f32 (0 where no labelled pixel), y_valid: [B, smax] u8 (y > 0); cnt_ws: [B, smax] f32 scratch.
int supervision_pool(const long long* seg, const float* mask, int batch, int channels, int h, int w, int smax, float* y,
                     unsigned char* y_valid, float* cnt_ws, cudaStream_t stream);

// Segment-wise maps: map[b, p] = v[b, seg[b, p]] for ids in [0, min(n_rows[b], smax)), NaN otherwise.  seg: [B, hw]
// int64 or int32; trav / conf: [B, smax] f32 (conf and conf_map may both be null); n_rows: [B] i32 on the device.
int segment_maps(const void* seg, bool seg_int64, int batch, long long hw, const float* trav, const float* conf, int smax,
                 const int* n_rows, float* trav_map, float* conf_map, cudaStream_t stream);

}  // namespace wvn
