/*
 * dva_conv2d.h -- C ABI of libdva_conv2d.so: the from-scratch image encoder (ResNetDown with
 * weight-standardised convolutions and GroupNorm) on the H100 (sm_90a).
 *
 * The entry points replace Conv2dWS, nn.Conv2d (1x1 downsample), nn.GroupNorm and ReLUWS of the
 * reference's torch_points3d/modules/multimodal/modalities/image.py:39-189 for the three convolution
 * shapes the shipped configs use.  libdva_conv2d.so links against libdva_b200.so (rpath $ORIGIN): it
 * reports its errors through dva_last_error() and counts its launches in dva_launch_count() of that library.
 *
 * Conventions: those of dva_b200.h (device pointers, sizes, the stream last, DVA_E* return codes: <0 = argument
 * error, nothing launched; >0 = cudaError_t of the failed launch).
 *   - every feature map is fp32, channels-last rows [B * H * W, C] (image-major, then row, then column);
 *   - products run on tensor cores in 3xTF32 (fp32-grade); nothing that is summed uses atomics: per-CTA
 *     partials are reduced in a fixed order, so every result is bitwise reproducible run to run;
 *   - GroupNorm statistics are per (image, group), over the C / G channels of the group and all pixels
 *     of the image, biased variance, as torch.nn.GroupNorm; C % G == 0.
 */
#ifndef DVA_CONV2D_H_
#define DVA_CONV2D_H_

#include "dva_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* convolution kinds: (kernel, stride, padding) */
enum {
  DVA_CONV_3X3_REFLECT = 0, /* 3x3, stride 1, reflect padding 1: H' = H, W' = W; needs H, W >= 2 */
  DVA_CONV_2X2_S2 = 1,      /* 2x2, stride 2, no padding: H' = H / 2, W' = W / 2 (floor) */
  DVA_CONV_1X1 = 2          /* 1x1, stride 1, no padding */
};

/* Filter preparation.  w [Co][Ci][R][S] (torch layout).  standardize = 1: per filter, subtract the mean over
 * Ci*R*S and divide by (unbiased std + 1e-5) * sqrt(Ci) (image.py:39-50, scaled=True); standardize = 0: copy.
 * Writes wf [Co][R][S][Ci] (the forward's K-major filter) and wd, the filter the data gradient reads:
 * [Ci][R][S][Co] for the 3x3 and 1x1 kinds, [R][S][Ci][Co] for the 2x2 kind. */
int dva_conv2d_weight_prep(const float* w, int Co, int Ci, int kind, int standardize, float* wf, float* wd,
                           void* stream);

/* Backward of the standardisation: dw [Co][Ci][R][S] from dwf, the gradient of wf ([Co][R][S][Ci]). */
int dva_conv2d_weight_prep_bwd(const float* w, const float* dwf, int Co, int Ci, int kind, float* dw, void* stream);

size_t dva_conv2d_fwd_workspace_bytes(int64_t B, int64_t Ho, int64_t Wo, int Co, int G);

/* z = conv(x, wf) + bias, x [B*H*W, Ci], z [B*Ho*Wo, Co]; and the GroupNorm statistics of z with G groups:
 * mean, invstd [B, G] (invstd = 1 / sqrt(var + eps)).  The per-CTA sums of z and z^2 are taken in the epilogue
 * in fp64 and reduced in a fixed order. */
int dva_conv2d_fwd(const float* x, int64_t B, int64_t H, int64_t W, int Ci, const float* wf, const float* bias,
                   int Co, int kind, int G, float eps, float* z, float* mean, float* invstd, void* ws,
                   size_t ws_bytes, void* stream);

/* dx = conv^T(dz, wd) (+ add, when add is not NULL; add may alias dx), dz [B*Ho*Wo, Co], dx [B*H*W, Ci].
 * 3x3 reflect: the mirrored taps are folded back onto rows / columns 1 and H-2 / W-2.  2x2: rows and columns
 * dropped by the floor get 0 (+ add). */
int dva_conv2d_dgrad(const float* dz, int64_t B, int64_t H, int64_t W, int Ci, int Co, const float* wd, int kind,
                     const float* add, float* dx, void* stream);

size_t dva_conv2d_wgrad_workspace_bytes(int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind);

/* dwf [Co][R][S][Ci] = sum over output pixels of dz x im2col(x), dbias [Co] = column sums of dz. */
int dva_conv2d_wgrad(const float* dz, const float* x, int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind,
                     float* dwf, float* dbias, void* ws, size_t ws_bytes, void* stream);

/* y = act(GN(z)) [+ skip] [+ GN_s(zs)], z / zs / skip / y [B*P, C]; GN(z) = (z - mean) * invstd * gamma + beta
 * with the statistics of (image, group); act = relu(.) * relu_scale when relu_scale > 0, the identity when
 * relu_scale == 0 (ReLUWS: relu_scale = sqrt(2 / (1 - 1/pi))).  skip and zs may be NULL. */
int dva_conv2d_gn_apply(const float* z, int64_t B, int64_t P, int C, int G, const float* mean, const float* invstd,
                        const float* gamma, const float* beta, float relu_scale, const float* skip, const float* zs,
                        const float* mean_s, const float* invstd_s, const float* gamma_s, const float* beta_s,
                        float* y, void* stream);

size_t dva_conv2d_gn_bwd_workspace_bytes(int64_t B, int64_t P, int C, int G);

/* Backward of one act(GN(z)) term of dva_conv2d_gn_apply: dz [B*P, C], dgamma, dbeta [C] from dy. */
int dva_conv2d_gn_bwd(const float* dy, const float* z, int64_t B, int64_t P, int C, int G, const float* mean,
                      const float* invstd, const float* gamma, const float* beta, float relu_scale, float* dz,
                      float* dgamma, float* dbeta, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* DVA_CONV2D_H_ */
