// getImages on the device (SURVEY 8f-1): ImageTransformer + image.scale fused into one HBM-bound kernel.
// Reference: ImageDetect.lua:22-52, modules/ImageTransformer.lua:19-33; the arithmetic lives in image_scale.cuh
// (shared with the CPU suite). One thread per output pixel of the 3 x h x w scaled image, x fastest so the store is
// coalesced; the 4 .. (f+2)^2 source reads of neighbouring threads overlap and are served by L1 / L2 (the raw image is
// a few MB, far below the 50 MB L2). Algorithmic bytes: 3*H0*W0*4 read + 3*h*w*4 written.
#include "common.cuh"
#include "image_scale.cuh"

// sx / sy: the two axis steps, divided once on the host (same IEEE division => same bits as the per-pixel division of the
// first version, which spent most of its ~300 instructions per pixel in three fdivs: 20.8 us for 480x640 -> 600x800)
__global__ void __launch_bounds__(256) get_images_kernel(mpn_img::TransformedImage I, int h, int w, float sx, float sy, float *__restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  const int c = blockIdx.z;
  if (x >= w) return;
  out[((int64_t)c * h + y) * w + x] = mpn_img::scaled_pixel(I, h, w, c, y, x, sx, sy);
}

// ImageDetect.lua:31-39: im_scale = scale / min(H0, W0), capped so that round(im_scale * max(H0, W0)) <= max_size;
// image.scale receives H0*im_scale, W0*im_scale as Lua numbers and allocates the result with them truncated to long.
int mpn_get_images_size_impl(int32_t H0, int32_t W0, double scale, double max_size, int32_t *h, int32_t *w, double *im_scale) {
  if (H0 <= 0 || W0 <= 0 || !(scale > 0) || !(max_size > 0)) return MPN_ERR_ARG;
  const double smin = H0 < W0 ? H0 : W0, smax = H0 < W0 ? W0 : H0;
  double s = scale / smin;
  if (floor(s * smax + 0.5) > max_size) s = max_size / smax;    // torch.round: half away from zero (positive here)
  if (h) *h = (int32_t)(long)((double)H0 * s);
  if (w) *w = (int32_t)(long)((double)W0 * s);
  if (im_scale) *im_scale = s;
  return MPN_OK;
}

static int get_images_launch_any(mpn_ctx *ctx, const float *im_dev, const uint8_t *im_u8_dev, int32_t H0, int32_t W0,
                                 const mpn_image_transform *tf, int32_t h, int32_t w, float *out_dev) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  MPN_CHECK_ARG(ctx, (im_dev || im_u8_dev) && out_dev && tf, "getImages: buffers missing");
  MPN_CHECK_ARG(ctx, H0 > 0 && W0 > 0 && h > 0 && w > 0 && h <= 65535, "getImages: bad sizes");
  mpn_img::TransformedImage I;
  I.im = im_dev; I.im_u8 = im_u8_dev; I.lut = nullptr; I.H0 = H0; I.W0 = W0;
  if (im_u8_dev) {     // byte -> float table: the 256 correctly rounded quotients b / 255.0f, divided once on the host (IEEE: same bits)
    if (!ctx->u8_lut_dev) {
      static float tab[256];
      static const bool init = [] { for (int b = 0; b < 256; ++b) tab[b] = (float)b / 255.0f; return true; }();
      (void)init;
      MPN_CUDA(ctx, cudaMalloc((void **)&ctx->u8_lut_dev, sizeof(tab)));
      MPN_CUDA(ctx, cudaMemcpyAsync(ctx->u8_lut_dev, tab, sizeof(tab), cudaMemcpyHostToDevice, ctx->stream));
    }
    I.lut = ctx->u8_lut_dev;
  }
  for (int c = 0; c < 3; ++c) {
    MPN_CHECK_ARG(ctx, tf->swap[c] >= 1 && tf->swap[c] <= 3, "ImageTransformer: swap entries are 1-based channel numbers");
    I.t.src_chan[c] = tf->swap[c] - 1;
    I.t.neg_mean[c] = (float)(-(double)tf->mean[c]);
    I.t.std[c] = tf->std[c];
  }
  I.t.has_scale = tf->scale != 1.0f;
  I.t.scale = tf->scale;
  I.t.has_std = tf->has_std != 0;
  dim3 grid((unsigned)((w + 255) / 256), (unsigned)h, 3);
  get_images_kernel<<<grid, 256, 0, ctx->stream>>>(I, h, w, mpn_img::axis_scale(W0, w), mpn_img::axis_scale(H0, h), out_dev);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}
int mpn_get_images_launch(mpn_ctx *ctx, const float *im_dev, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                          int32_t h, int32_t w, float *out_dev) {
  return get_images_launch_any(ctx, im_dev, nullptr, H0, W0, tf, h, w, out_dev);
}
int mpn_get_images_u8_launch(mpn_ctx *ctx, const uint8_t *im_hwc_dev, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                             int32_t h, int32_t w, float *out_dev) {
  return get_images_launch_any(ctx, nullptr, im_hwc_dev, H0, W0, tf, h, w, out_dev);
}
