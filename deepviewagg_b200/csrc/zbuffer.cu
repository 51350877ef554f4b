// Point -> pixel visibility: camera projection, splat boxes and the z-buffer.
//   reference (authoritative CPU/numba variants, README.md:122-123 says to avoid its own GPU
//   path): camera_projection_cpu visibility.py:478-538, equirectangular_projection_cpu :150-182,
//   equirectangular_splat_cpu :630-704, pinhole_splat_cpu :761-827,
//   visibility_from_splatting_cpu :1073-1195.
//
// z-buffer: the reference walks points in ascending order and overwrites a pixel iff
// dist < depth (strict), i.e. the winner of a pixel is argmin over (dist, index) in
// lexicographic order.  dist > 0 so its fp32 bit pattern is order-preserving as an unsigned
// integer; one 64-bit atomicMin on (dist_bits << 32 | index) per covered pixel realises exactly
// that order, independent of scheduling -> deterministic and bit-identical to the CPU loop.
// HBM-bound integer work: 8 B atomic per covered pixel; the [W,Hc] uint64 map (4 MB at
// 1024x512) lives in L2.
#include "dva_common.cuh"
#include "libm_f32.h"

namespace dva {

constexpr unsigned long long kEmpty = 0xffffffffffffffffull;

// ---- Z1: equirectangular projection ---------------------------------------------------------
// pose = [img_xyz(3), R(9 row-major)] fp32 on device; R = pose_to_rotation_matrix (host mirror).
// numba semantics reproduced: xyz, dist, v, t, p are float32; every expression that mixes a
// float32 array with a Python float (np.pi) is evaluated in float64 (that is why the reference
// returns float64 pixel coordinates, visibility.py:250-252).  Bit-exactness of the pixel indices
// needs two more facts, both measured on the executed reference (oracle/make_golden.py fixtures):
//  * `xyz_to_img.dot(rotation.transpose())` is a BLAS sgemm whose k-loop is a chain of fused
//    multiply-adds in k order: v = fma(dz, r2, fma(dy, r1, dx * r0));
//  * np.arctan2 / np.arccos on float32 are libm's atan2f / acosf, which are NOT correctly rounded;
//    libm_f32.h reproduces glibc's float-only evaluation operation by operation.
__global__ void __launch_bounds__(256)
project_equirect_kernel(const float* __restrict__ xyz, const float* __restrict__ pose,
                        float* __restrict__ dist, double* __restrict__ x_proj,
                        double* __restrict__ y_proj, uint8_t* __restrict__ keep, int64_t n,
                        int W, int H, int crop_top, int crop_bottom, float r_min, float r_max) {
  const float cx = pose[0], cy = pose[1], cz = pose[2];
  float R[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) R[j] = pose[3 + j];
  const double PI = 3.141592653589793;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float dx = xyz[3 * i] - cx, dy = xyz[3 * i + 1] - cy, dz = xyz[3 * i + 2] - cz;
    // norm_cpu: sqrt((v**2).sum(axis=1)) in float32, left-to-right
    const float d = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    dist[i] = d;
    // v = xyz_to_img . R^T (float32)
    const float v0 = __fmaf_rn(dz, R[2], __fmaf_rn(dy, R[1], __fmul_rn(dx, R[0])));
    const float v1 = __fmaf_rn(dz, R[5], __fmaf_rn(dy, R[4], __fmul_rn(dx, R[3])));
    const float v2 = __fmaf_rn(dz, R[8], __fmaf_rn(dy, R[7], __fmul_rn(dx, R[6])));
    const float t = dva_atan2f(v1, v0);
    const float p = dva_acosf(__fdiv_rn(v2, d));
    double w = ((double)(W - 1) * (1.0 - (double)t / PI) / 2.0);
    double h = ((double)(H - 1) * (double)p / PI);
    w = __dsub_rn(w, __dmul_rn(floor(w / (double)W), (double)W));   // numpy/python '%' (no DFMA contraction)
    h = __dsub_rn(h, __dmul_rn(floor(h / (double)H), (double)H));
    if (w != w) w = 0.0;
    if (h != h) h = 0.0;
    x_proj[i] = w; y_proj[i] = h;
    const bool in_range = (r_min < d) && (d < r_max);
    const bool in_fov = (0.0 <= w) && (w < (double)W) && ((double)crop_top <= h) &&
                        (h < (double)(H - crop_bottom));
    keep[i] = (in_range && in_fov) ? 1 : 0;
  }
}

// ---- Z1: pinhole / fisheye projection (visibility.py:219-339) --------------------------------
// cam = [img_xyz(3), A(9), t0(3), t1(3), intr(8)] fp32 on device, p = A (xyz - t0) + t1:
//   scannet               A = R(c2w), t0 = 0, t1 = T(c2w), c2w = inv(extrinsic)   (:233-236)
//   kitti360_{persp,fish}  A = R^T,    t0 = T, t1 = 0                              (:239-242, :305-308)
// camera 1: pinhole, intr = fx, fy, cx, cy (float32 arithmetic like numba, then float64)
// camera 3: fisheye, intr = xi, k1, k2, gamma1, gamma2, u0, v0 (float64 after the norm, like numba)
__global__ void __launch_bounds__(256)
project_camera_kernel(const float* __restrict__ xyz, const float* __restrict__ cam, int camera,
                      float* __restrict__ dist, double* __restrict__ x_proj,
                      double* __restrict__ y_proj, uint8_t* __restrict__ keep, int64_t n, int W, int H,
                      int crop_top, int crop_bottom, float r_min, float r_max) {
  float c[26];
#pragma unroll
  for (int j = 0; j < 26; ++j) c[j] = cam[j];
  const float* A = c + 3; const float* t0 = c + 12; const float* t1 = c + 15; const float* in = c + 18;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float px = xyz[3 * i], py = xyz[3 * i + 1], pz = xyz[3 * i + 2];
    const float dx = px - c[0], dy = py - c[1], dz = pz - c[2];
    const float d = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    dist[i] = d;
    const float q0 = px - t0[0], q1 = py - t0[1], q2 = pz - t0[2];
    // R @ xyz.T is an sgemm: fused multiply-add chain in k order (see project_equirect_kernel), then "+ T"
    const float p0 = __fadd_rn(__fmaf_rn(A[2], q2, __fmaf_rn(A[1], q1, __fmul_rn(A[0], q0))), t1[0]);
    const float p1 = __fadd_rn(__fmaf_rn(A[5], q2, __fmaf_rn(A[4], q1, __fmul_rn(A[3], q0))), t1[1]);
    const float p2 = __fadd_rn(__fmaf_rn(A[8], q2, __fmaf_rn(A[7], q1, __fmul_rn(A[6], q0))), t1[2]);
    double x, y, z;
    if (camera == 1) {
      x = (double)__fadd_rn(__fdiv_rn(__fmul_rn(p0, in[0]), p2), in[2]);
      y = (double)__fadd_rn(__fdiv_rn(__fmul_rn(p1, in[1]), p2), in[3]);
      z = (double)p2;
    } else {
      const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(p0, p0), __fmul_rn(p1, p1)), __fmul_rn(p2, p2)));
      // float64 like numba (visibility.py:323-336); every product / sum rounded on its own -- nvcc would
      // otherwise contract a * b + c into one DFMA, which LLVM (numba) and gcc -ffp-contract=off do not
      const double den = __dadd_rn((double)nrm, 1e-4);
      double fx = __ddiv_rn((double)p0, den), fy = __ddiv_rn((double)p1, den);
      const double fz = __ddiv_rn((double)p2, den);
      const double dz_ = __dadd_rn(fz, (double)in[0]);
      fx = __ddiv_rn(fx, dz_);
      fy = __ddiv_rn(fy, dz_);
      const double r2 = __dadd_rn(__dmul_rn(fx, fx), __dmul_rn(fy, fy)), r4 = __dmul_rn(r2, r2);
      const double poly = __dadd_rn(__dadd_rn(1.0, __dmul_rn((double)in[1], r2)), __dmul_rn((double)in[2], r4));
      x = __dadd_rn(__dmul_rn(__dmul_rn((double)in[3], poly), fx), (double)in[5]);
      y = __dadd_rn(__dmul_rn(__dmul_rn((double)in[4], poly), fy), (double)in[6]);
      z = __ddiv_rn((double)__fmul_rn(nrm, p2), fabs(__dadd_rn((double)p2, 1e-4)));
    }
    x_proj[i] = x; y_proj[i] = y;
    const bool in_range = (r_min < d) && (d < r_max);
    const bool in_fov = (0.0 <= x) && (x < (double)W) && ((double)crop_top <= y) &&
                        (y < (double)(H - crop_bottom)) && (0.0 < z);
    keep[i] = (in_range && in_fov) ? 1 : 0;
  }
}

// ---- Z2: splat boxes ------------------------------------------------------------------------
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__global__ void __launch_bounds__(256)
splat_boxes_kernel(const double* __restrict__ x_proj, const double* __restrict__ y_proj,
                   const float* __restrict__ dist, int32_t* __restrict__ splat, int64_t m, int W,
                   int H, int crop_top, int crop_bottom, double voxel, double k_swell,
                   double log_d_swell, int camera, double fx, double fy) {
  const double PI = 3.141592653589793;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m;
       i += (int64_t)gridDim.x * blockDim.x) {
    const double d = (double)dist[i];
    const double xp = x_proj[i], yp = y_proj[i];
    // (1 + k_swell * exp(-dist / log(d_swell))) * voxel / dist   (visibility.py:651-652, :783)
    const double swell = __dadd_rn(1.0, __dmul_rn(k_swell, exp(-d / log_d_swell))) * voxel / d;   // no DFMA contraction
    double wx, wy;
    if (camera == 0) {
      wy = swell * (double)H / PI;
      const double a = swell * (double)W / (2.0 * PI);
      const double b = PI / (double)H;
      wx = a / (sin(b * yp) + 0.001);
    } else {
      wx = swell * fx;
      wy = swell * fy;
    }
    // np.round -> half-to-even (rint), stored through float32 then int32 (:668-676)
    int xa = (int)(float)rint(xp - wx / 2.0);
    int xb = (int)(float)rint(xp + wx / 2.0 + 1.0);
    int ya = (int)(float)rint(yp - wy / 2.0);
    int yb = (int)(float)rint(yp + wy / 2.0 + 1.0);
    const int y_min = crop_top, y_max = H - crop_bottom;
    xa = clampi(xa, 0, W - 1);
    xb = clampi(xb, 1, W);
    ya = clampi(ya, y_min, y_max - 1);
    yb = clampi(yb, y_min + 1, y_max);
    reinterpret_cast<int4*>(splat)[i] = make_int4(xa, xb, ya, yb);
  }
}

// fisheye: the splat width comes from a second projection of the voxel top (visibility.py:903-914),
// computed by the host mirror; this kernel only rounds and clamps like the other cameras.
__global__ void __launch_bounds__(256)
splat_boxes_width_kernel(const double* __restrict__ x_proj, const double* __restrict__ y_proj,
                         const double* __restrict__ width, int32_t* __restrict__ splat, int64_t m,
                         int W, int H, int crop_top, int crop_bottom) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m;
       i += (int64_t)gridDim.x * blockDim.x) {
    const double xp = x_proj[i], yp = y_proj[i], w = width[i];
    int xa = (int)(float)rint(xp - w / 2.0);
    int xb = (int)(float)rint(xp + w / 2.0 + 1.0);
    int ya = (int)(float)rint(yp - w / 2.0);
    int yb = (int)(float)rint(yp + w / 2.0 + 1.0);
    const int y_min = crop_top, y_max = H - crop_bottom;
    reinterpret_cast<int4*>(splat)[i] = make_int4(clampi(xa, 0, W - 1), clampi(xb, 1, W),
                                                  clampi(ya, y_min, y_max - 1), clampi(yb, y_min + 1, y_max));
  }
}

// ---- Z3: z-buffer -----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
fill_u64_kernel(unsigned long long* __restrict__ p, unsigned long long v, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

constexpr int kLanesPerPoint = 8;   // typical splats cover 4..16 pixels

__global__ void __launch_bounds__(256)
zbuffer_raster_kernel(const int32_t* __restrict__ splat, const float* __restrict__ dist,
                      unsigned long long* __restrict__ zbuf, int64_t m, int Hc, int crop_top) {
  const int sub = threadIdx.x % kLanesPerPoint;
  const int64_t groups = ((int64_t)gridDim.x * blockDim.x) / kLanesPerPoint;
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / kLanesPerPoint; i < m; i += groups) {
    const int4 b = reinterpret_cast<const int4*>(splat)[i];
    const int xa = b.x, xb = b.y, ya = b.z - crop_top, yb = b.w - crop_top;
    const int hh = yb - ya, area = (xb - xa) * hh;
    const unsigned long long key =
        ((unsigned long long)__float_as_uint(dist[i]) << 32) | (unsigned long long)(uint32_t)i;
    for (int q = sub; q < area; q += kLanesPerPoint) {
      const int x = xa + q / hh, y = ya + q % hh;
      atomicMin(zbuf + (int64_t)x * Hc + y, key);
    }
  }
}

__global__ void __launch_bounds__(256)
zbuffer_resolve_kernel(const unsigned long long* __restrict__ zbuf, int64_t* __restrict__ idx_map,
                       uint8_t* __restrict__ seen, int64_t npix, int exact) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npix;
       i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = zbuf[i];
    if (exact) {
      idx_map[i] = -1;
      if (k != kEmpty) seen[(uint32_t)(k & 0xffffffffull)] = 1;
    } else {
      idx_map[i] = (k == kEmpty) ? (int64_t)-1 : (int64_t)(k & 0xffffffffull);
    }
  }
}

// exact mode: only splat centres of seen points; later (higher) index overwrites (:1183-1187)
__global__ void __launch_bounds__(256)
zbuffer_centres_kernel(const uint8_t* __restrict__ seen, const double* __restrict__ x_proj,
                       const double* __restrict__ y_proj, int64_t* __restrict__ idx_map,
                       int64_t m, int Hc, int crop_top) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (!seen[i]) continue;
    const int x = (int)x_proj[i];                 // astype(np.int32): truncation (:1177-1178)
    const int y = (int)y_proj[i] - crop_top;
    atomicMax(reinterpret_cast<long long*>(idx_map) + (int64_t)x * Hc + y, (long long)i);
  }
}

}  // namespace dva

using namespace dva;

extern "C" int dva_project_equirectangular(const float* xyz, const float* img_pose,
                                           float* dist, double* x_proj, double* y_proj,
                                           uint8_t* keep, int64_t n, int64_t W, int64_t H,
                                           int64_t crop_top, int64_t crop_bottom, float r_min,
                                           float r_max, void* stream) {
  if (n < 0 || W < 1 || H < 1 || crop_top < 0 || crop_bottom < 0 || crop_top + crop_bottom >= H)
    return fail(DVA_EINVAL, "project_equirectangular: bad sizes");
  if (n == 0) return DVA_OK;
  if (!xyz || !img_pose || !dist || !x_proj || !y_proj || !keep)
    return fail(DVA_EINVAL, "project_equirectangular: null pointer");
  project_equirect_kernel<<<grid_cap(n, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      xyz, img_pose, dist, x_proj, y_proj, keep, n, (int)W, (int)H, (int)crop_top,
      (int)crop_bottom, r_min, r_max);
  return check_launch("project_equirect");
}

extern "C" int dva_project_camera(const float* xyz, const float* cam, int camera, float* dist,
                                  double* x_proj, double* y_proj, uint8_t* keep, int64_t n, int64_t W,
                                  int64_t H, int64_t crop_top, int64_t crop_bottom, float r_min,
                                  float r_max, void* stream) {
  if (n < 0 || W < 1 || H < 1 || crop_top < 0 || crop_bottom < 0 || crop_top + crop_bottom >= H)
    return fail(DVA_EINVAL, "project_camera: bad sizes");
  if (camera != 1 && camera != 3) return fail(DVA_EUNSUPPORTED, "project_camera: camera must be 1 (pinhole) or 3 (fisheye)");
  if (n == 0) return DVA_OK;
  if (!xyz || !cam || !dist || !x_proj || !y_proj || !keep) return fail(DVA_EINVAL, "project_camera: null pointer");
  project_camera_kernel<<<grid_cap(n, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      xyz, cam, camera, dist, x_proj, y_proj, keep, n, (int)W, (int)H, (int)crop_top, (int)crop_bottom, r_min, r_max);
  return check_launch("project_camera");
}

extern "C" int dva_splat_boxes(const double* x_proj, const double* y_proj, const float* dist,
                               int32_t* splat, int64_t m, int64_t W, int64_t H, int64_t crop_top,
                               int64_t crop_bottom, double voxel, double k_swell, double d_swell,
                               int camera, double fx, double fy, void* stream) {
  if (m < 0 || W < 1 || H < 1 || crop_top < 0 || crop_bottom < 0 || crop_top + crop_bottom >= H)
    return fail(DVA_EINVAL, "splat_boxes: bad sizes");
  if (camera != 0 && camera != 1) return fail(DVA_EUNSUPPORTED, "splat_boxes: camera must be 0 (equirectangular) or 1 (pinhole)");
  if (m == 0) return DVA_OK;
  if (!x_proj || !y_proj || !dist || !splat) return fail(DVA_EINVAL, "splat_boxes: null pointer");
  if (!aligned16(splat)) return fail(DVA_EALIGN, "splat_boxes: splat must be 16-byte aligned");
  splat_boxes_kernel<<<grid_cap(m, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      x_proj, y_proj, dist, splat, m, (int)W, (int)H, (int)crop_top, (int)crop_bottom, voxel,
      k_swell, log(d_swell), camera, fx, fy);
  return check_launch("splat_boxes");
}

extern "C" int dva_splat_boxes_from_width(const double* x_proj, const double* y_proj,
                                          const double* width, int32_t* splat, int64_t m, int64_t W,
                                          int64_t H, int64_t crop_top, int64_t crop_bottom, void* stream) {
  if (m < 0 || W < 1 || H < 1 || crop_top < 0 || crop_bottom < 0 || crop_top + crop_bottom >= H)
    return fail(DVA_EINVAL, "splat_boxes_from_width: bad sizes");
  if (m == 0) return DVA_OK;
  if (!x_proj || !y_proj || !width || !splat) return fail(DVA_EINVAL, "splat_boxes_from_width: null pointer");
  if (!aligned16(splat)) return fail(DVA_EALIGN, "splat_boxes_from_width: splat must be 16-byte aligned");
  splat_boxes_width_kernel<<<grid_cap(m, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      x_proj, y_proj, width, splat, m, (int)W, (int)H, (int)crop_top, (int)crop_bottom);
  return check_launch("splat_boxes_from_width");
}

extern "C" int dva_zbuffer_splat(const int32_t* splat, const float* dist, const double* x_proj,
                                 const double* y_proj, unsigned long long* zbuf, int64_t* idx_map,
                                 uint8_t* seen, int64_t m, int64_t W, int64_t H,
                                 int64_t crop_top, int64_t crop_bottom, int exact, void* stream) {
  if (m < 0 || W < 1 || H < 1 || crop_top < 0 || crop_bottom < 0 || crop_top + crop_bottom >= H)
    return fail(DVA_EINVAL, "zbuffer_splat: bad sizes");
  if (m >= (1ll << 32)) return fail(DVA_EUNSUPPORTED, "zbuffer_splat: more than 2^32 points");
  if (!zbuf || !idx_map || (m > 0 && (!splat || !dist))) return fail(DVA_EINVAL, "zbuffer_splat: null pointer");
  if (exact && m > 0 && (!seen || !x_proj || !y_proj)) return fail(DVA_EINVAL, "zbuffer_splat: exact mode needs seen/x_proj/y_proj");
  if (m > 0 && !aligned16(splat)) return fail(DVA_EALIGN, "zbuffer_splat: splat must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t Hc = H - crop_top - crop_bottom, npix = W * Hc;
  fill_u64_kernel<<<grid_cap(npix, 256, 16), 256, 0, st>>>(zbuf, kEmpty, npix);
  int rc = check_launch("zbuffer_fill");
  if (rc) return rc;
  if (exact && m > 0) {
    cudaError_t e = cudaMemsetAsync(seen, 0, (size_t)m, st);
    if (e != cudaSuccess) return fail((int)e, "zbuffer_splat: memset failed");
  }
  if (m > 0) {
    zbuffer_raster_kernel<<<grid_cap(m * kLanesPerPoint, 256, 16), 256, 0, st>>>(splat, dist, zbuf, m, (int)Hc, (int)crop_top);
    rc = check_launch("zbuffer_raster");
    if (rc) return rc;
  }
  zbuffer_resolve_kernel<<<grid_cap(npix, 256, 16), 256, 0, st>>>(zbuf, idx_map, seen, npix, exact);
  rc = check_launch("zbuffer_resolve");
  if (rc) return rc;
  if (exact && m > 0) {
    zbuffer_centres_kernel<<<grid_cap(m, 256, 16), 256, 0, st>>>(seen, x_proj, y_proj, idx_map, m, (int)Hc, (int)crop_top);
    rc = check_launch("zbuffer_centres");
  }
  return rc;
}
