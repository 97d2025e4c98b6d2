// sampling.cuh -- bilinear image sampling shared by the kernels that read the rgb views.
#pragma once

#include <stdint.h>

namespace b2 {

// mve::Image<uint8_t>::linear_at on one channel of the interleaved rgb image
__device__ __forceinline__ uint8_t linear_at_rgb(const uint8_t *__restrict__ img, int w, int h, float x, float y, int ch)
{
    x = fmaxf(0.0f, fminf((float)(w - 1), x));
    y = fmaxf(0.0f, fminf((float)(h - 1), y));
    int fx = (int)x, fy = (int)y;
    int fx1 = min(fx + 1, w - 1), fy1 = min(fy + 1, h - 1);
    float w1 = x - (float)fx, w0 = 1.0f - w1;
    float w3 = y - (float)fy, w2 = 1.0f - w3;
    float r = (float)img[3 * (fx + (size_t)fy * w) + ch] * (w0 * w2) + (float)img[3 * (fx1 + (size_t)fy * w) + ch] * (w1 * w2)
        + (float)img[3 * (fx + (size_t)fy1 * w) + ch] * (w0 * w3) + (float)img[3 * (fx1 + (size_t)fy1 * w) + ch] * (w1 * w3) + 0.5f;
    return (uint8_t)r;
}

}  // namespace b2
