/*
 * dva_resnet.h -- C ABI of libdva_resnet.so: the ResNet-18 image encoders on the H100 (sm_90a) -- the dilated one
 * pretrained on ADE20K (mit_semseg's resnet18dilated behind the reference's ADE20KResNet18* wrappers), torchvision's
 * ImageNet one (ResNet18*) and the Cityscapes one (CityscapesResNet18*): zero-padded convolutions with the BatchNorm
 * statistics in their epilogue, train- and eval-mode BatchNorm (also synchronised over ranks), the 3x3 stride-2 max
 * pools (padding 1 or 0) and the bilinear resize of the wrappers (align_corners=False).
 *
 * libdva_resnet.so links against libdva_b200.so (rpath $ORIGIN): it reports its errors through dva_last_error() and
 * counts its launches in dva_launch_count() of that library.
 *
 * Conventions: fp32 channels-last rows [B * H * W, C]; products in 3xTF32 on tensor cores (the main loop of
 * libdva_conv2d.so); no atomics: every result is bitwise reproducible run to run; the stream last; DVA_E* return
 * codes.  A convolution is (T, stride, dilation) with zero padding = dilation * (T - 1) / 2 and no bias; the shapes
 * are those of the trunks: 3x3 stride 1 with dilation 1, 2 or 4, 3x3 stride 2 with dilation 1, 1x1 with stride 1
 * or 2, and the ImageNet stem's 7x7 stride 2 (padding 3).  Its output is H' = (H - 1) / stride + 1 (ceil(H / stride)).
 */
#ifndef DVA_RESNET_H_
#define DVA_RESNET_H_

#include "dva_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* w [Co][Ci][T][T] (the torch layout) -> wf [Co][T][T][Ci] (the forward's operand) and wd [Ci][T][T][Co] (the data
 * gradient's). */
int dva_resnet_weight_prep(const float* w, int Co, int Ci, int T, float* wf, float* wd, void* stream);

size_t dva_resnet_fwd_workspace_bytes(int64_t B, int64_t Ho, int64_t Wo, int Co);

/* z = conv(x, wf), x [B*H*W, Ci], z [B*H'*W', Co], followed by the BatchNorm statistics of z (F.batch_norm on one
 * device).  training != 0: the epilogue takes fp64 per-(64-row tile, channel) sums of z and z^2; they are reduced in
 * tile order to mean and invstd = 1 / sqrt(biased var + eps), and running_mean / running_var are updated in place
 * with `momentum` (running_var with the unbiased variance).  training == 0: mean = running_mean, invstd =
 * 1 / sqrt(running_var + eps); the running stats are read only and ws may be NULL. */
int dva_resnet_conv_bn_fwd(const float* x, int64_t B, int64_t H, int64_t W, int Ci, const float* wf, int Co, int T,
                           int stride, int dil, int training, float momentum, float eps, float* running_mean,
                           float* running_var, float* z, float* mean, float* invstd, void* ws, size_t ws_bytes,
                           void* stream);

/* Training-mode BatchNorm synchronised over ranks (nn.SyncBatchNorm), the forward in two calls around one
 * all-reduce of `sums` (fp64 [2 * C + 1]: per channel (sum z, sum z^2), then the count):
 *   dva_resnet_conv_bn_fwd_sums: z = conv(x, wf) as dva_resnet_conv_bn_fwd does it, and this rank's sums, reduced in
 *     tile order as there, with the count B*H'*W' (one value per channel is allowed here);
 *   dva_resnet_bn_sync_stats: from the all-reduced sums and the global count n (>= 2, else DVA_EINVAL), mean, invstd
 *     and the running-stat update with `momentum` (running_var with the unbiased variance of n values).
 * Over the sums of one rank with its own count, the results are those of dva_resnet_conv_bn_fwd bit for bit. */
int dva_resnet_conv_bn_fwd_sums(const float* x, int64_t B, int64_t H, int64_t W, int Ci, const float* wf, int Co,
                                int T, int stride, int dil, float* z, double* sums, void* ws, size_t ws_bytes,
                                void* stream);
int dva_resnet_bn_sync_stats(const double* sums, int C, int64_t n, float momentum, float eps, float* running_mean,
                             float* running_var, float* mean, float* invstd, void* stream);

/* dx [B*H*W, Ci] = the data gradient of conv for dz [B*H'*W', Co] (+ add when add is not NULL; add may alias dx). */
int dva_resnet_conv_dgrad(const float* dz, int64_t B, int64_t H, int64_t W, int Ci, int Co, const float* wd, int T,
                          int stride, int dil, const float* add, float* dx, void* stream);

size_t dva_resnet_wgrad_workspace_bytes(int64_t B, int64_t H, int64_t W, int Ci, int Co, int T, int stride, int dil);

/* dw [Co][Ci][T][T] (the torch layout) = sum over output pixels of dz x taps of x; split over the pixels, the fp32
 * split partials summed in fp64 in split order. */
int dva_resnet_conv_wgrad(const float* dz, const float* x, int64_t B, int64_t H, int64_t W, int Ci, int Co, int T,
                          int stride, int dil, float* dw, void* ws, size_t ws_bytes, void* stream);

/* y = relu(BN(z) [+ skip] [+ BN_s(zs)]) over [M, C], BN(z) = (z - mean) * invstd * gamma + beta per channel. */
int dva_resnet_bn_apply(const float* z, int64_t M, int C, const float* mean, const float* invstd, const float* gamma,
                        const float* beta, const float* skip, const float* zs, const float* mean_s,
                        const float* invstd_s, const float* gamma_s, const float* beta_s, float* y, void* stream);

size_t dva_resnet_bn_bwd_workspace_bytes(int64_t M, int C);

/* Backward of y = relu(BN(z) + r): g = dy where y > 0, 0 elsewhere; per-channel sums of g and g * zhat in fp64 over
 * pixel chunks, reduced in chunk order: dbeta, dgamma; dz = gamma * invstd * (g - mean(g) - zhat * mean(g * zhat))
 * (training) or gamma * invstd * g (eval).  g is written to gout when it is not NULL (the gradient of r). */
int dva_resnet_bn_bwd(const float* dy, const float* y, const float* z, int64_t M, int C, const float* mean,
                      const float* invstd, const float* gamma, int training, float* dz, float* gout, float* dgamma,
                      float* dbeta, void* ws, size_t ws_bytes, void* stream);

/* The backward of a synchronised BatchNorm in two calls around one all-reduce of `sums` (fp64 [2 * C + 1]: per
 * channel (sum g, sum g * zhat), then the count):
 *   dva_resnet_bn_bwd_sums: this rank's sums, reduced in chunk order as in dva_resnet_bn_bwd, with the count M, and
 *     this rank's dbeta, dgamma (the gradient all-reduce sums them over ranks); ws as dva_resnet_bn_bwd's;
 *   dva_resnet_bn_sync_bwd: from the all-reduced sums and the global count n (>= max(M, 2)), dz = gamma * invstd *
 *     (g - sum g / n - zhat * sum (g * zhat) / n) and g to gout when it is not NULL; ws holds C * 16 bytes.
 * Over the sums of one rank with its own count, the results are those of dva_resnet_bn_bwd bit for bit. */
int dva_resnet_bn_bwd_sums(const float* dy, const float* y, const float* z, int64_t M, int C, const float* mean,
                           const float* invstd, float* dgamma, float* dbeta, double* sums, void* ws, size_t ws_bytes,
                           void* stream);
int dva_resnet_bn_sync_bwd(const float* dy, const float* y, const float* z, int64_t M, int C, const float* mean,
                           const float* invstd, const float* gamma, const double* sums, int64_t n, float* dz,
                           float* gout, void* ws, size_t ws_bytes, void* stream);

/* MaxPool2d(3, stride 2, padding pad), pad 0 or 1: y [B*H'*W', C], H' = (H + 2 pad - 3) / 2 + 1, and the window
 * position (r * 3 + s) of the max: the first valid tap starts as the max and a later one replaces it when greater or
 * NaN (torch's rule), so padding never wins.  H + 2 pad < 3 (no window) is DVA_EINVAL.  The backward sums, for each
 * input pixel, the at most 4 windows that chose it; a pixel no window covers (the last row or column at pad 0) gets
 * 0. */
int dva_resnet_maxpool_pad(const float* x, int64_t B, int64_t H, int64_t W, int C, int pad, float* y, uint8_t* arg,
                           void* stream);
int dva_resnet_maxpool_pad_bwd(const float* dy, const uint8_t* arg, int64_t B, int64_t H, int64_t W, int C, int pad,
                               float* dx, void* stream);
/* The same with padding 1, H' = (H - 1) / 2 + 1. */
int dva_resnet_maxpool(const float* x, int64_t B, int64_t H, int64_t W, int C, float* y, uint8_t* arg, void* stream);
int dva_resnet_maxpool_bwd(const float* dy, const uint8_t* arg, int64_t B, int64_t H, int64_t W, int C, float* dx,
                           void* stream);

/* Bilinear resize, align_corners=False, of x [B*H*W, C] to Ho x Wo, written to columns [col0, col0 + C) of rows of
 * ldy floats: the source index of output o is max(scale * (o + 0.5) - 0.5, 0), scale = 1 / scale_factor or in / out
 * as torch computes it (passed in).  The backward gathers, for each input pixel, the output pixels that read it. */
int dva_resnet_resize(const float* x, int64_t B, int64_t H, int64_t W, int C, int64_t Ho, int64_t Wo, float scale_h,
                      float scale_w, float* y, int64_t ldy, int64_t col0, void* stream);
int dva_resnet_resize_bwd(const float* dy, int64_t ldy, int64_t col0, int64_t B, int64_t H, int64_t W, int C,
                          int64_t Ho, int64_t Wo, float scale_h, float scale_w, float* dx, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* DVA_RESNET_H_ */
