"""Point -> pixel visibility on the GPU, with the reference's function / class names
(torch_points3d/core/multimodal/visibility.py).  Results follow the reference's CPU (numba)
variants, which are the authoritative ones (its README.md:122-123 warns against its own GPU
mapping path): integer outputs -- splat boxes, z-buffer winners, pixel coordinates -- are
bit-identical to the numba loops given the same projections.

  camera_projection          <- visibility.py:478-538, 592-623   (equirectangular, pinhole, fisheye)
  visibility_from_splatting  <- visibility.py:1073-1195, 1288-1322
  postprocess_features       <- visibility.py:1548-1582
  read_s3dis_depth_map       <- visibility.py:1328-1358            (host, PIL)
  visibility_from_depth_map  <- visibility.py:1361-1392
  k_nn_image_system          <- visibility.py:1396-1460
  visibility_biasutti        <- visibility.py:1463-1500
  VisibilityModel, SplattingVisibility, DepthBasedVisibility, BiasuttiVisibility
                             <- visibility.py:1677-1799

Kernels: csrc/zbuffer.cu through the C ABI (dva_project_equirectangular, dva_project_camera,
dva_splat_boxes, dva_splat_boxes_from_width, dva_zbuffer_splat) and the exact grid k-NN of
csrc/knn_features.cu (mapping.knn_grid) for the image-plane neighbours of the Biasutti model.
Compaction of the kept set / winner map is index plumbing (torch.nonzero); the Biasutti
contrast and the depth-map test are O(n k) / O(n) gathers and comparisons in torch.
"""
import numpy as np
import torch

from ..._lib import launch, require_cuda

_PINHOLE_CAMERAS = ("scannet", "kitti360_perspective")


def pose_to_rotation_matrix(opk):
    """Rotation matrix of an (omega, phi, kappa) pose: M_o . (M_p . M_k), float32 -- the
    arithmetic of pose_to_rotation_matrix_cpu (visibility.py:57-90), done on the host."""
    opk = np.asarray(opk.detach().cpu().numpy() if isinstance(opk, torch.Tensor) else opk, dtype=np.float32)
    co, so = np.cos(opk[0]), np.sin(opk[0])
    cp, sp = np.cos(opk[1]), np.sin(opk[1])
    ck, sk = np.cos(opk[2]), np.sin(opk[2])
    m_o = np.array([[1.0, 0.0, 0.0], [0.0, co, -so], [0.0, so, co]], dtype=np.float32)
    m_p = np.array([[cp, 0.0, sp], [0.0, 1.0, 0.0], [-sp, 0.0, cp]], dtype=np.float32)
    m_k = np.array([[ck, -sk, 0.0], [sk, ck, 0.0], [0.0, 0.0, 1.0]], dtype=np.float32)
    return torch.from_numpy(np.dot(m_o, np.dot(m_p, m_k)).astype(np.float32))


def _inv4_f32(E):
    """float32 inverse of the 4x4 extrinsic exactly as numba's np.linalg.inv computes it
    (visibility.py:233): LAPACK sgetrf + sgetri (numpy's own inv solves against the identity with
    sgesv instead and differs in the last bit, which moves ~40 % of the float pixel coordinates
    by one ulp).  Host-side camera set-up, once per image."""
    try:
        from scipy.linalg import lapack
    except ImportError as e:  # pragma: no cover - scipy ships with the image (numba needs it too)
        raise ImportError("the 'scannet' camera needs scipy's LAPACK bindings for a bit-exact "
                          "camera-to-world matrix") from e
    lu, piv, info = lapack.sgetrf(E)
    if info != 0:
        raise np.linalg.LinAlgError("singular extrinsic matrix")
    inv, info = lapack.sgetri(lu, piv)
    if info != 0:
        raise np.linalg.LinAlgError("singular extrinsic matrix")
    return np.ascontiguousarray(inv, dtype=np.float32)


def _camera_transform(camera, img_extrinsic):
    """(A, t0, t1) float32 with p = A (xyz - t0) + t1 (visibility.py:231-244, 304-310)."""
    E = np.ascontiguousarray(np.asarray(
        img_extrinsic.detach().cpu().numpy() if isinstance(img_extrinsic, torch.Tensor) else img_extrinsic,
        dtype=np.float32))
    if camera == 'scannet':
        c2w = _inv4_f32(E)
        return c2w[:3, :3].copy(), np.zeros(3, np.float32), c2w[:3, 3].copy()
    return E[:3, :3].T.copy(), E[:3, 3].copy(), np.zeros(3, np.float32)


def _host_f32(t, n):
    t = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return np.asarray(t, dtype=np.float32).reshape(-1)[:n]


def camera_projection(xyz, img_xyz, img_opk=None, img_intrinsic_pinhole=None, img_intrinsic_fisheye=None,
                      img_extrinsic=None, img_mask=None, img_size=(1024, 512), crop_top=0, crop_bottom=0,
                      r_max=30, r_min=0.5, camera='s3dis_equirectangular', **kwargs):
    """-> (indices int64[m], dist f32[m], x_proj f64[m], y_proj f64[m]) of the points within
    (r_min, r_max) of the camera that project inside the (cropped) image and its mask
    (visibility.py:478-538).  Cameras: s3dis_equirectangular, scannet, kitti360_perspective,
    kitti360_fisheye."""
    require_cuda(xyz)
    dev = xyz.device
    xyz = xyz.float().contiguous()
    n = xyz.shape[0]
    W, H = int(img_size[0]), int(img_size[1])
    dist = torch.empty(n, dtype=torch.float32, device=dev)
    x_proj = torch.empty(n, dtype=torch.float64, device=dev)
    y_proj = torch.empty(n, dtype=torch.float64, device=dev)
    keep = torch.empty(n, dtype=torch.uint8, device=dev)
    cam_xyz = _host_f32(img_xyz, 3)
    if camera == 's3dis_equirectangular':
        rot = pose_to_rotation_matrix(img_opk if img_opk is not None else np.zeros(3, np.float32))
        pose = torch.from_numpy(np.concatenate([cam_xyz, rot.numpy().reshape(-1)])).to(dev)
        launch("dva_project_equirectangular", dev, xyz, pose, dist, x_proj, y_proj, keep, n, W, H, int(crop_top),
               int(crop_bottom), float(r_min), float(r_max))
    elif camera in _PINHOLE_CAMERAS or camera == 'kitti360_fisheye':
        A, t0, t1 = _camera_transform(camera, img_extrinsic)
        intr = np.zeros(8, np.float32)
        if camera == 'kitti360_fisheye':
            intr[:7] = _host_f32(img_intrinsic_fisheye, 7)
            code = 3
        else:
            K = img_intrinsic_pinhole.detach().cpu().numpy() if isinstance(img_intrinsic_pinhole, torch.Tensor) \
                else np.asarray(img_intrinsic_pinhole)
            K = np.asarray(K, dtype=np.float32)
            intr[:4] = [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]
            code = 1
        cam = torch.from_numpy(np.concatenate([cam_xyz, A.reshape(-1), t0, t1, intr]).astype(np.float32)).to(dev)
        launch("dva_project_camera", dev, xyz, cam, code, dist, x_proj, y_proj, keep, n, W, H, int(crop_top),
               int(crop_bottom), float(r_min), float(r_max))
    else:
        raise ValueError(f"unknown camera '{camera}'")
    if img_mask is not None:  # field_of_view_cpu: img_mask[floor(x), floor(y)] (visibility.py:428-434)
        assert tuple(img_mask.shape) == (W, H), \
            f'Expected img_mask to be a torch.BoolTensor of shape img_size={img_size} but got size={img_mask.shape}.'
        xi = x_proj.floor().long().clamp(0, W - 1)
        yi = y_proj.floor().long().clamp(0, H - 1)
        keep = keep.bool() & img_mask.to(dev)[xi, yi]
    indices = torch.nonzero(keep, as_tuple=False).view(-1)
    return indices, dist[indices], x_proj[indices], y_proj[indices]


def _project_raw(xyz, camera, img_extrinsic, intr8, code):
    """x_proj, y_proj of every row of xyz (no filtering) through dva_project_camera."""
    dev, n = xyz.device, xyz.shape[0]
    A, t0, t1 = _camera_transform(camera, img_extrinsic)
    cam = torch.from_numpy(np.concatenate([np.zeros(3, np.float32), A.reshape(-1), t0, t1, intr8])
                           .astype(np.float32)).to(dev)
    d = torch.empty(n, dtype=torch.float32, device=dev)
    xp = torch.empty(n, dtype=torch.float64, device=dev)
    yp = torch.empty(n, dtype=torch.float64, device=dev)
    keep = torch.empty(n, dtype=torch.uint8, device=dev)
    launch("dva_project_camera", dev, xyz, cam, code, d, xp, yp, keep, n, 1 << 20, 1 << 20, 0, 0, 0.0, 1e30)
    return xp, yp


def fisheye_splat_boxes(x_proj, y_proj, xyz, img_extrinsic, img_intrinsic_fisheye, img_size=(1024, 512),
                        crop_top=0, crop_bottom=0, voxel=0.02, k_swell=1.0, d_swell=1000,
                        camera='kitti360_fisheye'):
    """fisheye_splat_cpu (visibility.py:876-953): the splat width is twice the image distance between
    a point and the projection of the top of its voxel (xyz + [0, 0, swell * voxel / 2]); NB the
    reference takes `dist = norm(xyz)` of the ABSOLUTE coordinates here (:900), reproduced."""
    require_cuda(x_proj, y_proj, xyz)
    xyz = xyz.float().contiguous()
    m = xyz.shape[0]
    # norm_cpu: float32, squares summed left to right (a device-side reduction may associate otherwise)
    d = torch.sqrt((xyz[:, 0] * xyz[:, 0] + xyz[:, 1] * xyz[:, 1]) + xyz[:, 2] * xyz[:, 2])
    swell = 1 + k_swell * torch.exp(-d.double() / np.log(d_swell))          # float64, like numba
    top = xyz.clone()
    top[:, 2] += (swell * voxel / 2).float()                                # z_offset is float32
    intr = np.zeros(8, np.float32)
    intr[:7] = _host_f32(img_intrinsic_fisheye, 7)
    xt, yt = _project_raw(top, camera, img_extrinsic, intr, 3)
    width = 2 * torch.sqrt((x_proj.double() - xt) ** 2 + (y_proj.double() - yt) ** 2)
    splat = torch.empty((m, 4), dtype=torch.int32, device=xyz.device)
    launch("dva_splat_boxes_from_width", xyz.device, x_proj.double().contiguous(), y_proj.double().contiguous(),
           width.contiguous(), splat, m, int(img_size[0]), int(img_size[1]), int(crop_top), int(crop_bottom))
    return splat


def splat_boxes(x_proj, y_proj, dist, img_intrinsic_pinhole=None, img_size=(1024, 512), crop_top=0,
                crop_bottom=0, voxel=0.02, k_swell=1.0, d_swell=1000, camera='s3dis_equirectangular'):
    """[m,4] int32 (x_a, x_b, y_a, y_b) like *_splat_cpu (visibility.py:630-704, 761-827)."""
    require_cuda(x_proj, y_proj, dist)
    m = x_proj.shape[0]
    splat = torch.empty((m, 4), dtype=torch.int32, device=x_proj.device)
    if camera == 's3dis_equirectangular':
        cam, fx, fy = 0, 0.0, 0.0
    elif camera in _PINHOLE_CAMERAS:
        cam = 1
        fx, fy = float(img_intrinsic_pinhole[0][0]), float(img_intrinsic_pinhole[1][1])
    else:
        raise NotImplementedError(f"camera='{camera}' has no CUDA splat kernel yet")
    launch("dva_splat_boxes", x_proj.device, x_proj.double().contiguous(), y_proj.double().contiguous(),
           dist.float().contiguous(), splat, m, int(img_size[0]), int(img_size[1]), int(crop_top), int(crop_bottom),
           float(voxel), float(k_swell), float(d_swell), cam, fx, fy)
    return splat


def visibility_from_splatting(x_proj, y_proj, dist, xyz=None, img_extrinsic=None, img_intrinsic_pinhole=None,
                              img_intrinsic_fisheye=None, img_size=(1024, 512), crop_top=0, crop_bottom=0,
                              voxel=0.1, k_swell=1.0, d_swell=1000, exact=False,
                              camera='s3dis_equirectangular', **kwargs):
    """Z-buffer visibility -> (indices, x_pix, y_pix) in the reference's order (row-major over the
    [x, y] winner map).  Ties go to the lowest point index; `exact` keeps splat centres only."""
    require_cuda(x_proj, y_proj, dist)
    assert x_proj.shape[0] == y_proj.shape[0] == dist.shape[0] > 0
    dev = x_proj.device
    W, H = int(img_size[0]), int(img_size[1])
    Hc = H - int(crop_top) - int(crop_bottom)
    xp, yp = x_proj.double().contiguous(), y_proj.double().contiguous()
    d = dist.float().contiguous()
    m = d.shape[0]
    if camera == 'kitti360_fisheye':
        splat = fisheye_splat_boxes(xp, yp, xyz, img_extrinsic, img_intrinsic_fisheye, img_size, crop_top,
                                    crop_bottom, voxel, k_swell, d_swell, camera)
    else:
        splat = splat_boxes(xp, yp, d, img_intrinsic_pinhole, img_size, crop_top, crop_bottom, voxel, k_swell,
                            d_swell, camera)
    zbuf = torch.empty(W * Hc, dtype=torch.int64, device=dev)       # uint64 keys
    idx_map = torch.empty((W, Hc), dtype=torch.int64, device=dev)
    seen = torch.empty(m, dtype=torch.uint8, device=dev) if exact else None
    launch("dva_zbuffer_splat", dev, splat, d, xp, yp, zbuf, idx_map, seen, m, W, H, int(crop_top), int(crop_bottom),
           int(bool(exact)))
    pix = torch.nonzero(idx_map >= 0, as_tuple=False)
    x_pix, y_pix = pix[:, 0], pix[:, 1]
    return idx_map[x_pix, y_pix], x_pix, y_pix + int(crop_top)


# -------------------------------------------------------------------------------------------------
# depth-map visibility
# -------------------------------------------------------------------------------------------------
def read_s3dis_depth_map(path, img_size=None, empty=-1):
    """S3DIS depth PNG (16 bit, 1/512 m per unit, 65535 = no depth) -> float32 [W, H] CPU tensor
    in metres, `empty` where there is no depth (visibility.py:1328-1358).  `img_size` = (W, H)
    resizes with nearest-neighbour sampling first."""
    from PIL import Image
    im = Image.open(path)
    if img_size is not None:
        im = im.resize(tuple(int(v) for v in img_size), resample=Image.NEAREST)
    a = np.array(im).T
    out = a.astype(np.float32) / np.float32(512)        # exact: v < 2**16, 512 a power of two
    out[a == 2 ** 16 - 1] = empty
    return torch.from_numpy(np.ascontiguousarray(out))


def visibility_from_depth_map(x_proj, y_proj, dist, depth_map_path=None, img_size=(1024, 512),
                              depth_threshold=0.05, depth_map=None, **kwargs):
    """Points whose depth is within `depth_threshold` of the depth map at their pixel
    -> (indices, x_proj, y_proj) of the kept points, ascending (visibility.py:1361-1392).
    `depth_map` ([W, H] float32) is used as is; otherwise the S3DIS PNG at `depth_map_path` is read
    at `img_size`.  The comparison is |d_real - dist| <= depth_threshold in float32 (torch
    compares an fp32 tensor with a Python float in fp32)."""
    require_cuda(x_proj, y_proj, dist)
    assert x_proj.shape[0] == y_proj.shape[0] == dist.shape[0] > 0
    if depth_map is None:
        assert depth_map_path is not None, 'Please provide depth_map_path or depth_map.'
        depth_map = read_s3dis_depth_map(depth_map_path, img_size=img_size, empty=-1)
    depth_map = depth_map.to(x_proj.device, torch.float32)
    dist_real = depth_map[x_proj.long(), y_proj.long()]
    thr = torch.tensor(depth_threshold, dtype=torch.float32, device=x_proj.device)
    indices = torch.nonzero((dist_real - dist.float()).abs() <= thr, as_tuple=False).view(-1)
    return indices, x_proj[indices], y_proj[indices]


# -------------------------------------------------------------------------------------------------
# Biasutti visibility
# -------------------------------------------------------------------------------------------------
def k_nn_image_system(x_proj, y_proj, k=75, x_margin=None, x_width=None):
    """[n, k'] int64: the k nearest projections of every projection in the image plane, self
    included, k' = min(k, search-set size) (visibility.py:1396-1460).  With `x_margin` > 0 and
    `x_width` > 0 the image wraps around in x: the search set is the n projections, then copies of
    those with x <= x_margin shifted by +x_width, then copies of those with x >= x_width - x_margin
    shifted by -x_width; copies are reported as their original index.  Exact search on the GPU grid
    k-NN (the reference runs a brute-force KeOps argKmin): squared distance dx*dx + dy*dy in fp32,
    ties by search-set index."""
    from .mapping import knn_grid
    require_cuda(x_proj, y_proj)
    assert x_margin is None or x_width > 0, 'x_margin and x_width must both be provided for image wrapping.'
    n = x_proj.shape[0]
    xy = torch.stack((x_proj.float(), y_proj.float()), dim=1)
    wrap_x = x_margin is not None and x_margin > 0 and x_width is not None and x_width > 0
    if wrap_x:
        off = torch.tensor([[float(np.float32(x_width)), 0.0]], dtype=torch.float32, device=xy.device)
        idx_left = torch.nonzero(x_proj <= x_margin, as_tuple=False).view(-1)
        idx_right = torch.nonzero(x_proj >= (x_width - x_margin), as_tuple=False).view(-1)
        search = torch.cat((xy, xy[idx_left] + off, xy[idx_right] - off))
    else:
        search = xy
    m = search.shape[0]
    kk = min(int(k), m)
    pos = torch.cat((search, torch.zeros((m, 1), dtype=torch.float32, device=xy.device)), dim=1)
    neighbors = knn_grid(pos, kk)[:n]
    if wrap_x and m > n:
        orig = torch.cat((torch.arange(n, device=xy.device), idx_left, idx_right))
        neighbors = orig[neighbors]
    return neighbors


def visibility_biasutti(x_proj, y_proj, dist, img_size=None, k=75, margin=None, threshold=None, **kwargs):
    """Biasutti et al., "Visibility estimation in point clouds with variable density"
    (visibility.py:1463-1500): alpha = exp(-((d - d_min) / (d_max - d_min))**2) over the k
    image-plane neighbours, kept where alpha >= threshold -> (indices, x_proj, y_proj) ascending.
    `threshold=None` is the mean of alpha, summed in float64 and rounded to float32 (the reference
    takes a float32 mean, a few ulps away).  A point whose neighbours all share one depth gets
    alpha = NaN (0/0) and is never kept; with the mean threshold, one NaN keeps nothing."""
    require_cuda(x_proj, y_proj, dist)
    assert x_proj.shape[0] == y_proj.shape[0] == dist.shape[0] > 0
    neighbors = k_nn_image_system(x_proj, y_proj, k=k, x_margin=margin, x_width=img_size[0])
    d = dist.float()
    dist_nn = d[neighbors]
    dist_min = dist_nn.min(dim=1).values
    dist_max = dist_nn.max(dim=1).values
    alpha = torch.exp(-((d - dist_min) / (dist_max - dist_min)) ** 2)
    if threshold is None:
        thr = alpha.double().mean().float()
    else:
        thr = torch.tensor(threshold, dtype=torch.float32, device=alpha.device)
    indices = torch.nonzero(alpha >= thr, as_tuple=False).view(-1)
    return indices, x_proj[indices], y_proj[indices]


def postprocess_features(xyz_to_img, y_proj, dist, linearity, planarity, scattering, normals,
                         img_size=(1024, 512), r_max=30, r_min=0.5, **kwargs):
    """[n,F] viewing-condition features (visibility.py:1548-1582): normalised depth, linearity,
    planarity, scattering, |cos(view, normal)|, normalised pixel height."""
    features = []
    if dist is not None:
        # tensor / tensor: a CUDA division by a Python scalar is evaluated as a multiplication by its
        # reciprocal (1 ulp off the reference's CPU result, normalize_dist_cuda visibility.py:1503-1518)
        d = dist.float()
        features.append(((d - r_min) / torch.full_like(d, r_max + 1e-4)).float())
    for f in (linearity, planarity, scattering):
        if f is not None:
            features.append(f)
    if xyz_to_img is not None and dist is not None and normals is not None:
        u = (xyz_to_img / (dist + 1e-4).reshape((-1, 1))).float()
        p = u * normals.float()
        features.append(((p[:, 0] + p[:, 1]) + p[:, 2]).abs())           # torch CPU's sum order over 3 terms
    if y_proj is not None:
        features.append((y_proj / torch.full_like(y_proj, float(img_size[1]))).float())
    return torch.stack(features).t()


class VisibilityModel:
    """Same call contract as the reference's VisibilityModel (visibility.py:1677-1761)."""

    def __init__(self, img_size=(1024, 512), crop_top=0, crop_bottom=0, r_max=30, r_min=0.5,
                 camera='s3dis_equirectangular'):
        self.img_size = img_size
        self.crop_top = crop_top
        self.crop_bottom = crop_bottom
        self.r_max = r_max
        self.r_min = r_min
        self.camera = camera

    def _camera_projection(self, *args, **kwargs):
        return camera_projection(*args, **self.__dict__, **kwargs)

    def _visibility(self, *args, **kwargs):
        raise NotImplementedError

    def _postprocess_features(self, *args):
        return postprocess_features(*args, **self.__dict__)

    def __call__(self, xyz, img_xyz, linearity=None, planarity=None, scattering=None, normals=None, **kwargs):
        dev = xyz.device
        idx_1, dist, x_proj, y_proj = self._camera_projection(xyz, img_xyz, **kwargs)
        if x_proj.shape[0] == 0:
            e_long = torch.empty((0,), dtype=torch.long, device=dev)
            e_f = torch.empty((0,), dtype=torch.float, device=dev)
            return {'idx': e_long, 'x': e_long.clone(), 'y': e_long.clone(), 'depth': e_f, 'features': e_f.clone()}
        idx_2, x_pix, y_pix = self._visibility(x_proj, y_proj, dist, xyz[idx_1], **kwargs)
        idx = idx_1[idx_2]
        dist, y_proj = dist[idx_2], y_proj[idx_2]
        out = {'idx': idx, 'x': x_pix, 'y': y_pix, 'depth': dist}
        pick = lambda t: t[idx] if t is not None else None  # noqa: E731
        img_xyz_d = torch.as_tensor(img_xyz, dtype=xyz.dtype, device=dev)
        out['features'] = self._postprocess_features(xyz[idx] - img_xyz_d, y_proj, dist, pick(linearity),
                                                     pick(planarity), pick(scattering), pick(normals))
        return out

    def __repr__(self):
        return f"{self.__class__.__name__}({', '.join(f'{k}={v}' for k, v in self.__dict__.items())})"


class SplattingVisibility(VisibilityModel):
    """visibility.py:1764-1776."""

    def __init__(self, voxel=0.1, k_swell=1.0, d_swell=1000, exact=False, **kwargs):
        super().__init__(**kwargs)
        self.voxel = voxel
        self.k_swell = k_swell
        self.d_swell = d_swell
        self.exact = exact

    def _visibility(self, x_proj, y_proj, dist, xyz, **kwargs):
        return visibility_from_splatting(x_proj, y_proj, dist, xyz, **self.__dict__, **kwargs)


class DepthBasedVisibility(VisibilityModel):
    """visibility.py:1779-1787.  The depth map comes per call: `depth_map` ([W, H] float32
    tensor) or `depth_map_path` (S3DIS PNG)."""

    def __init__(self, depth_threshold=0.05, **kwargs):
        super().__init__(**kwargs)
        self.depth_threshold = depth_threshold

    def _visibility(self, x_proj, y_proj, dist, xyz, **kwargs):
        return visibility_from_depth_map(x_proj, y_proj, dist, **self.__dict__, **kwargs)


class BiasuttiVisibility(VisibilityModel):
    """visibility.py:1790-1799."""

    def __init__(self, k=75, margin=None, threshold=None, **kwargs):
        super().__init__(**kwargs)
        self.k = k
        self.margin = margin
        self.threshold = threshold

    def _visibility(self, x_proj, y_proj, dist, xyz, **kwargs):
        return visibility_biasutti(x_proj, y_proj, dist, **self.__dict__, **kwargs)
