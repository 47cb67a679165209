// Internal: cv2.remap() restated on the device (image_transforms.cu), shared by transform_image() and match_feature().
#pragma once
#include <cuda_runtime.h>

namespace mb200 {

// out[Ho][Wo][channels] = src sampled at map[Ho][Wo][2] (float32), as cv2.remap() computes it. Device pointers; src's
// rows are stride bytes apart, the map and the output are packed. type: MRCAL_B200_IMAGE_*; interpolation:
// MRCAL_B200_INTER_*; border: MRCAL_B200_BORDER_*. Enqueued on s; false + set_error() if the launch fails
bool launch_remap(const void* src, size_t stride, int W, int H, const float* map, int Wo, int Ho, int type, int channels,
                  int interpolation, int border, const double* border_value, void* dst, cudaStream_t s);

}  // namespace mb200
