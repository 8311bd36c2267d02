// prep_image.cuh -- the per-pixel arithmetic of the input pipeline, shared by sb_prep_image (misc.cu) and
// sb_prep_stereo_pair (train_input.cu).
// Input pipeline (SURVEY 8f-3): prep_im_for_blob (lib/model/utils/blob.py:44-64) + HWC->CHW (demo.py:124-128):
// uint8 BGR image -> fp32 (pixel - PIXEL_MEANS) -> cv2.resize(fx=fy=scale, INTER_LINEAR) -> [3,Ho,Wo].
// OpenCV's separable fp32 bilinear restated: source coordinate (d+0.5)/scale-0.5 and its fraction in fp64, the
// horizontal pass on the two source rows first, then the vertical pass, one rounding per multiply / add.
#pragma once
#include "common.cuh"

struct ResizeTap { int i0, i1; float w0, w1; };
__device__ __forceinline__ ResizeTap resize_tap(int d, int n_src, double inv) {
    const double x = ((double)d + 0.5) * inv - 0.5;
    int s = (int)floor(x);
    float f = (float)(x - (double)s);
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= n_src - 1) { f = 0.f; s = n_src - 1; }
    ResizeTap t;
    t.i0 = s; t.i1 = min(s + 1, n_src - 1);
    t.w0 = __fsub_rn(1.0f, f); t.w1 = f;
    return t;
}

// output pixel (x, y) of all three channels.  mirror: read source column W-1-c where the unmirrored image would read
// column c, i.e. the prep of img[:, ::-1, :] (minibatch.py:117-118) without materialising it.
__device__ __forceinline__ void prep_pixel(const uint8_t* __restrict__ img, int H, int W, double inv, int rgb,
                                           int mirror, float* __restrict__ out, int Ho, int Wo, int x, int y) {
    const ResizeTap tx = resize_tap(x, W, inv), ty = resize_tap(y, H, inv);
    const int c0 = mirror ? W - 1 - tx.i0 : tx.i0, c1 = mirror ? W - 1 - tx.i1 : tx.i1;
    const double means[3] = {102.9801, 115.9465, 122.7717};        // cfg.PIXEL_MEANS (config.py:170), BGR
    const uint8_t* r0 = img + (size_t)ty.i0 * W * 3;
    const uint8_t* r1 = img + (size_t)ty.i1 * W * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int cs = rgb ? 2 - c : c;                            // demo.py:106-107: rgb -> bgr
        const float p00 = (float)((double)r0[c0 * 3 + cs] - means[c]), p01 = (float)((double)r0[c1 * 3 + cs] - means[c]);
        const float p10 = (float)((double)r1[c0 * 3 + cs] - means[c]), p11 = (float)((double)r1[c1 * 3 + cs] - means[c]);
        const float h0 = __fadd_rn(__fmul_rn(p00, tx.w0), __fmul_rn(p01, tx.w1));
        const float h1 = __fadd_rn(__fmul_rn(p10, tx.w0), __fmul_rn(p11, tx.w1));
        out[((size_t)c * Ho + y) * Wo + x] = __fadd_rn(__fmul_rn(h0, ty.w0), __fmul_rn(h1, ty.w1));
    }
}
