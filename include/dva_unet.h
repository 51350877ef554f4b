/*
 * dva_unet.h -- C ABI of libdva_unet.so: the transposed convolutions of the from-scratch image decoder
 * (ResNetUp with weight-standardised ConvTranspose2dWS and GroupNorm, and UnaryConv's activation) on the
 * H100 (sm_90a).
 *
 * The entry points replace ConvTranspose2dWS of the reference's torch_points3d/modules/multimodal/modalities/
 * image.py:76-107 for the two shapes the shipped configs use.  GroupNorm apply and backward, ReLUWS, the residual
 * and the 1x1 convolutions run on libdva_conv2d.so (include/dva_conv2d.h).  libdva_unet.so links against
 * libdva_b200.so (rpath $ORIGIN): it reports its errors through dva_last_error() and counts its launches in
 * dva_launch_count() of that library.
 *
 * Conventions: those of dva_conv2d.h (fp32 channels-last rows [B * H * W, C]; products in 3xTF32 on tensor cores;
 * no atomics: every result is bitwise reproducible run to run; the stream last; DVA_E* return codes).
 */
#ifndef DVA_UNET_H_
#define DVA_UNET_H_

#include "dva_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* transposed convolution kinds: (kernel, stride, padding), zero padding, output_padding 0 */
enum {
  DVA_UNET_UP_2X2 = 0,  /* 2x2, stride 2, padding 0: H' = 2 H, W' = 2 W */
  DVA_UNET_T_3X3 = 1    /* 3x3, stride 1, padding 1: H' = H, W' = W (a 3x3 zero-padded convolution with the
                           flipped, transposed filter) */
};

/* Filter preparation.  w [Ci][Co][R][S] (the torch layout of ConvTranspose2d).  Per input channel, subtract the
 * mean over Co*R*S and divide by (unbiased std + 1e-5) * sqrt(Co) (standardize_weights of image.py:39-50 on a
 * transposed weight: weight.shape[1] = Co, its square root in float32).  Writes the operands the GEMMs read:
 *   DVA_UNET_UP_2X2  wf [R][S][Co][Ci] (forward: [B*H*W, Ci] x [Ci, 4 Co]), wd [Ci][R][S][Co] (data gradient);
 *   DVA_UNET_T_3X3   wf [Co][R][S][Ci] with wf[o][ky][kx][c] = w^[c][o][2-ky][2-kx], wd [Ci][R][S][Co] unflipped. */
int dva_unet_weight_prep(const float* w, int Ci, int Co, int kind, float* wf, float* wd, void* stream);

/* Backward of the standardisation: dw [Ci][Co][R][S] from dwf, the gradient of wf (its layout). */
int dva_unet_weight_prep_bwd(const float* w, const float* dwf, int Ci, int Co, int kind, float* dw, void* stream);

size_t dva_unet_fwd_workspace_bytes(int64_t B, int64_t H, int64_t W, int Co, int G, int kind);

/* z = convT(x, wf) + bias, x [B*H*W, Ci], z [B*H'*W', Co]; and the GroupNorm statistics of z with G groups
 * (G <= 128): mean, invstd [B, G] (invstd = 1 / sqrt(var + eps)), from fp64 partial sums taken in the epilogue
 * and reduced in a fixed order.  H, W >= 1. */
int dva_unet_fwd(const float* x, int64_t B, int64_t H, int64_t W, int Ci, const float* wf, const float* bias, int Co,
                 int kind, int G, float eps, float* z, float* mean, float* invstd, void* ws, size_t ws_bytes,
                 void* stream);

/* dx = the data gradient of convT (+ add, when add is not NULL; add may alias dx), dz [B*H'*W', Co],
 * dx [B*H*W, Ci]: a 2x2 stride-2 convolution of dz (DVA_UNET_UP_2X2) or a zero-padded 3x3 one (DVA_UNET_T_3X3). */
int dva_unet_dgrad(const float* dz, int64_t B, int64_t H, int64_t W, int Ci, int Co, const float* wd, int kind,
                   const float* add, float* dx, void* stream);

size_t dva_unet_wgrad_workspace_bytes(int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind);

/* dwf (the layout of wf) = sum over pixels of dz x x, dbias [Co] = column sums of dz; split over the pixels, the
 * fp32 split partials summed in fp64 in split order. */
int dva_unet_wgrad(const float* dz, const float* x, int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind,
                   float* dwf, float* dbias, void* ws, size_t ws_bytes, void* stream);

/* y = relu(z) * scale over n elements (UnaryConv's activation: scale 1 for ReLU, sqrt(2 / (1 - 1/pi)) for
 * ReLUWS), and its backward dz = dy * scale where z > 0, 0 elsewhere. */
int dva_unet_act(const float* z, int64_t n, float scale, float* y, void* stream);
int dva_unet_act_bwd(const float* dy, const float* z, int64_t n, float scale, float* dz, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* DVA_UNET_H_ */
