// wvn-b200: internal interface of resnet_kernels.cu (the non-GEMM kernels of the ResNet backbone and its pooling).
#pragma once

#include <cuda_runtime.h>

namespace wvn {

// Convolution operand rows from an NHWC bf16 activation [batch, h, w, c] (c % 8 == 0): row (b, oy, ox) of `out` holds
// the k x k window at (oy * stride - pad, ox * stride - pad) in (ky, kx, channel) order, zero outside the map; rows are
// `pitch` elements apart and columns [k * k * c, pitch) are not written.
int im2col_nhwc(const void* in, int batch, int h, int w, int c, int k, int stride, int pad, void* out, long long pitch,
                cudaStream_t stream);
// The stem's rows straight from the fp32 NCHW image [batch, 3, h, w]: ImageNet Normalize first, then the zero padding,
// (ky, kx, channel) order as above; columns [k * k * 3, pitch) are not written.
int im2col_image(const float* img, int batch, int h, int w, int k, int stride, int pad, void* out, long long pitch,
                 cudaStream_t stream);
// 3 x 3 / stride 2 / pad 1 max-pool of an NHWC bf16 map [batch, h, w, c] (c % 8 == 0); padding is -inf.
int maxpool3s2_nhwc(const void* in, int batch, int h, int w, int c, void* out, cudaStream_t stream);

constexpr int kPyramidMaxLevels = 5;

struct PyramidArgs {
  int batch = 0, h = 0, w = 0, smax = 0;
  int levels = 0;                             // 1 .. kPyramidMaxLevels
  const void* taps[kPyramidMaxLevels] = {};  // NHWC bf16 [batch, th, tw, tp]; channels [tc, tp) are not read
  int th[kPyramidMaxLevels] = {}, tw[kPyramidMaxLevels] = {}, tc[kPyramidMaxLevels] = {}, tp[kPyramidMaxLevels] = {};
};
// out [batch, smax, sum(tc)] fp32: per segment, the mean of each level's cells whose nearest-downsampled id is the
// segment, levels concatenated; a segment without a cell at a level takes the cell under its full-resolution centroid
// (centers [batch, smax, 2] = (col, row)); a segment without pixels (NaN centroid) gets a NaN row.
int segment_pool_pyramid(const long long* seg, const float* centers, const PyramidArgs& a, float* out,
                         cudaStream_t stream);

}  // namespace wvn
