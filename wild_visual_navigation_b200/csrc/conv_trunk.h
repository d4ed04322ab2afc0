// wvn-b200: the convolutional trunk handles (wvn_resnet_*, wvn_effnet_*) — internal interface of conv_trunk.cu.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include "../../include/wvn_b200.h"

namespace wvn {

// taps: the trunk's feature levels, NHWC bf16 (4 for a ResNet, 5 for EfficientNet-B0).
int resnet_create(const wvn_resnet_config* cfg, wvn_resnet** out);
void resnet_destroy(wvn_resnet* h);
size_t resnet_workspace_bytes(const wvn_resnet* h);
int resnet_set_weight(wvn_resnet* h, const char* name, const float* data, long long numel);
int resnet_forward(wvn_resnet* h, const float* img, int batch, void* const* taps, cudaStream_t s);

int effnet_create(const wvn_effnet_config* cfg, wvn_effnet** out);
void effnet_destroy(wvn_effnet* h);
size_t effnet_workspace_bytes(const wvn_effnet* h);
int effnet_set_weight(wvn_effnet* h, const char* name, const float* data, long long numel);
int effnet_forward(wvn_effnet* h, const float* img, int batch, void* const* taps, cudaStream_t s);

}  // namespace wvn
