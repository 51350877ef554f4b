"""Point -> image mapping construction (the reference's MapImages transform,
torch_points3d/core/data_transform/multimodal/image.py:162-428) on the GPU kernels.

For every image of a SameSettingImageData: range filter + camera projection + splat z-buffer
(core/multimodal/visibility.py) -> pixel coordinates at the mapping resolution
(`// proj_upscale`, `- crop_offsets`, in-crop filter, `// downscale`, :307-319) -> duplicate
(point, px, py) removed (:328) -> one ImageMapping.from_dense over all images (:415-417), images no
point sees are dropped (:392-394).  The reference's per-image KD-tree sphere sampling (:242-245)
only pre-filters points by distance, which the projection kernel does itself (r_min < d < r_max),
so it has no counterpart here.  Tensors in, tensors out: the torch_geometric `Data` holder of the
reference is not needed on this path.
"""
import torch

from ...utils.multimodal import lexargunique, lexunique
from . import visibility as visibility_module
from .image import ImageMapping, SameSettingImageData


_METHODS = ('SplattingVisibility', 'DepthBasedVisibility', 'BiasuttiVisibility')


class MapImages:
    """`method` names the visibility model: 'SplattingVisibility' (z-buffer of splats),
    'BiasuttiVisibility' (depth contrast among the k nearest projections) or
    'DepthBasedVisibility' (agreement with a depth map: image i reads
    `images.extras['depth_map'][i]`, a [W_proj, H_proj] float32 map in metres, -1 where empty,
    e.g. from read_s3dis_depth_map)."""

    def __init__(self, method='SplattingVisibility', proj_upscale=None, ref_size=None, use_cuda=True,
                 verbose=False, cylinder=False, **kwargs):
        if not use_cuda:
            raise RuntimeError("deepviewagg_b200.MapImages runs on CUDA only (no CPU fallback)")
        if method not in _METHODS:
            raise NotImplementedError(f"unknown visibility method '{method}', expected one of {_METHODS}")
        self.method, self.proj_upscale, self.ref_size = method, proj_upscale, ref_size
        self.verbose, self.cylinder, self.kwargs = verbose, cylinder, kwargs

    def __call__(self, pos, images: SameSettingImageData, mapping_index=None, linearity=None, planarity=None,
                 scattering=None, normals=None, device='cuda'):
        """pos [N,3]; images: poses in `images.pos` / `images.opk` or `images.extras['extrinsic']`
        (+ 'intrinsic_pinhole' [B,4,4] / 'intrinsic_fisheye' [B,7]); returns a copy of `images`
        restricted to the seen images, with `.mappings` set."""
        assert images.num_views >= 1, "At least one image must be provided."
        if self.ref_size is not None:
            images.ref_size = tuple(self.ref_size)
            images.crop_size = images.ref_size
        if self.proj_upscale is not None:
            images.proj_upscale = self.proj_upscale
        proj_size = images.proj_size
        if images.mask is not None:      # points projecting onto a masked pixel neither map nor occlude
            assert tuple(images.mask.shape) == proj_size
        model = getattr(visibility_module, self.method)(img_size=proj_size, **self.kwargs)
        dev = torch.device(device)
        pos_d = pos.float().to(dev)
        n_points = pos.shape[0]
        ids = torch.arange(n_points, device=dev) if mapping_index is None else mapping_index.to(dev).long()
        to_d = lambda t: t.to(dev) if t is not None else None  # noqa: E731
        lin, pla, sca, nor = to_d(linearity), to_d(planarity), to_d(scattering), to_d(normals)
        ex = images.extras
        crop_off = images.crop_offsets if images.crop_offsets is not None else \
            torch.zeros((images.num_views, 2), dtype=torch.long)
        if self.method == 'DepthBasedVisibility':
            if 'depth_map' not in ex:
                raise ValueError("MapImages(method='DepthBasedVisibility') needs images.extras['depth_map'], a "
                                 "[B, W_proj, H_proj] float32 tensor of depth maps at the projection size "
                                 "(read_s3dis_depth_map(path, img_size=...) reads an S3DIS depth PNG)")
            dm = ex['depth_map']
            if tuple(dm.shape) != (images.num_views,) + proj_size:
                raise ValueError(f"images.extras['depth_map'] has shape {tuple(dm.shape)}, expected "
                                 f"{(images.num_views,) + proj_size} (one [W_proj, H_proj] map per image)")
        image_ids, point_ids, features, pixels = [], [], [], []
        for i in range(images.num_views):
            kw = {}
            if self.method == 'DepthBasedVisibility':
                kw['depth_map'] = ex['depth_map'][i].to(dev, torch.float32)
            if images.opk is not None:
                kw['img_opk'] = images.opk[i].float()
            if 'extrinsic' in ex:
                kw['img_extrinsic'] = ex['extrinsic'][i].float()
            if 'intrinsic_pinhole' in ex:
                kw['img_intrinsic_pinhole'] = ex['intrinsic_pinhole'][i].float()
            if 'intrinsic_fisheye' in ex:
                kw['img_intrinsic_fisheye'] = ex['intrinsic_fisheye'][i].float()
            if images.mask is not None:
                kw['img_mask'] = images.mask.to(dev)
            out = model(pos_d, images.pos[i].float(), linearity=lin, planarity=pla, scattering=sca, normals=nor,
                        **kw)
            if out['idx'].shape[0] == 0:
                continue
            pid = ids[out['idx']]
            px = out['x'].long() // images.proj_upscale - int(crop_off[i, 0])
            py = out['y'].long() // images.proj_upscale - int(crop_off[i, 1])
            inside = torch.where((px >= 0) & (py >= 0) & (px < images.crop_size[0]) & (py < images.crop_size[1]))[0]
            px = (px[inside] // images.downscale).long()
            py = (py[inside] // images.downscale).long()
            pid, feat = pid[inside], out['features'].float()[inside]
            keep = lexargunique(pid, px, py)
            image_ids.append(i)
            point_ids.append(pid[keep])
            features.append(feat[keep])
            pixels.append(torch.stack((px[keep], py[keep]), dim=1).to(images.pixel_dtype))
        if len(image_ids) == 0:
            raise ValueError(
                "No mappings were found between the 3D points and any of the provided images. Make sure your "
                "images are located in the vicinity of your point cloud and that the projection parameters "
                "allow for at least one point-image-pixel mapping.")
        seen = torch.tensor(image_ids, dtype=torch.long)
        out_images = images[seen]                      # unseen images dropped, the rest renumbered
        new_ids = torch.arange(len(image_ids), device=dev).repeat_interleave(
            torch.tensor([p.shape[0] for p in point_ids], device=dev))
        n_total = int(ids.max().item()) + 1
        out_images.mappings = ImageMapping.from_dense(torch.cat(point_ids), new_ids, torch.cat(pixels),
                                                      torch.cat(features), num_points=n_total)
        out_images.visibility = model
        return out_images


# ------------------------------------------------------------------------------------------------
# neighbourhood-based mapping features (density, occlusion)
# ------------------------------------------------------------------------------------------------
_MAX_CELLS = 1 << 26


def _grid_for(pos, cell_size):
    lo = pos.min(dim=0).values
    hi = pos.max(dim=0).values
    lo_l, hi_l = [float(v) for v in lo], [float(v) for v in hi]
    while True:
        dims = [max(1, int((h - l) / cell_size) + 1) for l, h in zip(lo_l, hi_l)]
        if dims[0] * dims[1] * dims[2] <= _MAX_CELLS:
            return lo_l, dims, cell_size
        cell_size *= 1.26


def _knn_search_grid(pos, k, cell_size=None):
    """Uniform grid over the search set `pos` [n,3] fp32 (CUDA, contiguous) shared by knn_grid and
    knn_query: returns (lo, dims, cell_size, cell_s, order, cell_ptr, xyz_s), the points sorted by
    cell, order[j] = original index of sorted slot j, cell_ptr [gx*gy*gz+1]."""
    from ..._lib import launch
    from .csr import pointers_from_sorted
    n = pos.shape[0]
    cell = torch.empty(n, dtype=torch.int64, device=pos.device)

    def assign(cs):
        lo, dims, cs = _grid_for(pos, cs)
        launch("dva_knn_cell_ids", pos.device, pos, cell, n, lo[0], lo[1], lo[2], cs, dims[0], dims[1], dims[2])
        return lo, dims, cs

    if cell_size is None:
        # start from a volume-uniform guess, then steer towards ~k/6 points per occupied cell
        # (scans are mostly surfaces: occupancy grows with the square of the cell size)
        target = max(2.0, k / 6)
        ext = pos.max(dim=0).values - pos.min(dim=0).values
        live = ext > 0
        dims_live = int(live.sum())
        if dims_live == 3:
            cell_size = float((ext.clamp_min(1e-6).prod() * k / n) ** (1 / 3))
        elif dims_live > 0:
            # planar (image-plane, z = 0) or collinear set: uniform over the axes that have extent,
            # ~target points per cell
            cell_size = float((ext[live].clamp_min(1e-6).prod() * target / n) ** (1 / dims_live))
        else:
            cell_size = 1.0                                 # all points coincide: one cell
        for _ in range(3):
            lo, dims, cell_size = assign(cell_size)
            per_cell = n / max(1, int(torch.unique(cell).numel()))
            if 0.5 * target <= per_cell <= 2 * target:
                break
            cell_size *= float((target / per_cell) ** 0.5)
    lo, dims, cell_size = assign(cell_size)
    cell_s, order = torch.sort(cell, stable=True)
    cell_ptr = pointers_from_sorted(cell_s, dims[0] * dims[1] * dims[2])
    xyz_s = pos[order].contiguous()
    return lo, dims, cell_size, cell_s, order, cell_ptr, xyz_s


def knn_grid(pos, k, cell_size=None, return_dist2=False):
    """Exact k nearest neighbours (self included, 1 <= k <= 128) of every point among all points,
    on CUDA (replaces the KeOps `argKmin` of image.py:504-514 and visibility.py:1439-1444).
    Squared distances are (dx*dx + dy*dy) + dz*dz in fp32, ties ordered by point index; points
    with z = 0 give the exact 2D distance (image-plane search).  Returns neighbors [N,k] int64
    (ascending distance) and optionally the squared distances."""
    from ..._lib import launch
    if not pos.is_cuda:
        raise RuntimeError("knn_grid runs on CUDA tensors only (no CPU fallback)")
    pos = pos.float().contiguous()
    n = pos.shape[0]
    if not 1 <= k <= 128:
        raise ValueError("knn_grid: k must be in [1, 128]")
    if n < k:
        raise ValueError(f"knn_grid: need at least k={k} points, got {n}")
    lo, dims, cell_size, cell_s, order, cell_ptr, xyz_s = _knn_search_grid(pos, k, cell_size)
    nbr = torch.empty((n, k), dtype=torch.int64, device=pos.device)
    d2 = torch.empty((n, k), dtype=torch.float32, device=pos.device) if return_dist2 else None
    launch("dva_knn_grid", pos.device, xyz_s, cell_s, order, cell_ptr, n, k, lo[0], lo[1], lo[2], cell_size, dims[0],
           dims[1], dims[2], nbr, d2)
    return (nbr, d2) if return_dist2 else nbr


_KNN_BLOCK = 8      # fine cells per coarse block and axis (csrc/knn_features.cu kKnnBlk)


def knn_query(query, search, k, cell_size=None, return_dist2=False):
    """Exact k nearest neighbours (1 <= k <= 128) of every point of `query` [M,3] among the points
    of `search` [n,3], on CUDA (replaces the KeOps brute-force `argmin` of
    models/segmentation/multimodal/no3d.py:105-125).  Same arithmetic and tie order as knn_grid:
    (dx*dx + dy*dy) + dz*dz in fp32, ties to the lower search index; knn_query(p, p, k) equals
    knn_grid(p, k).  The grid is built over the search set; a query far from every search point
    walks a coarse level of 8^3-cell blocks that skips empty space, so it never scans the whole
    set.  Returns neighbors [M,k] int64 (search indices, ascending distance) and optionally the
    squared distances."""
    from ..._lib import launch
    if not (query.is_cuda and search.is_cuda):
        raise RuntimeError("knn_query runs on CUDA tensors only (no CPU fallback)")
    if query.device != search.device:
        raise RuntimeError("knn_query: query and search must live on the same device")
    if not 1 <= k <= 128:
        raise ValueError("knn_query: k must be in [1, 128]")
    search = search.float().contiguous()
    query = query.float().contiguous()
    m, n = query.shape[0], search.shape[0]
    nbr = torch.empty((m, k), dtype=torch.int64, device=query.device)
    d2 = torch.empty((m, k), dtype=torch.float32, device=query.device) if return_dist2 else None
    if m == 0:
        return (nbr, d2) if return_dist2 else nbr
    if n < k:
        raise ValueError(f"knn_query: need at least k={k} search points, got {n}")
    lo, dims, cell_size, _, order, cell_ptr, xyz_s = _knn_search_grid(search, k, cell_size)
    gx, gy, gz = dims
    B = _KNN_BLOCK
    counts = (cell_ptr[1:] - cell_ptr[:-1]).view(gz, gy, gx)
    counts = torch.nn.functional.pad(counts, (0, (-gx) % B, 0, (-gy) % B, 0, (-gz) % B))
    GZ, GY, GX = counts.shape[0] // B, counts.shape[1] // B, counts.shape[2] // B
    blocks = counts.view(GZ, B, GY, B, GX, B).sum(dim=(1, 3, 5)).to(torch.int32).contiguous()
    qcell = torch.empty(m, dtype=torch.int64, device=query.device)
    launch("dva_knn_cell_ids", query.device, query, qcell, m, lo[0], lo[1], lo[2], cell_size, gx, gy, gz)
    qcell_s, qorder = torch.sort(qcell, stable=True)
    q_s = query[qorder].contiguous()
    launch("dva_knn_query", query.device, q_s, qcell_s, qorder, m, xyz_s, order, cell_ptr, blocks, n, k, lo[0], lo[1],
           lo[2], cell_size, gx, gy, gz, nbr, d2)
    return (nbr, d2) if return_dist2 else nbr


class NeighborhoodBasedMappingFeatures:
    """Append density and occlusion to the mapping features (the reference transform of the same
    name, core/data_transform/multimodal/image.py:431-612): for every k of `k` (int or list),
    density of each view's point from the radius of its k-NN ball, and occlusion = share of the
    point's k-NN (itself included) that the view's image also sees.  Columns: densities for
    ascending k, then occlusions for ascending k (:548-553, :590-600).

    `use_faiss` / `ncells` / `nprobes` are accepted for configuration compatibility; the search
    is always the exact one (the reference's KeOps branch)."""

    def __init__(self, k=20, voxel=None, density=True, occlusion=True, use_cuda=True, use_faiss=False,
                 ncells=None, nprobes=10, verbose=False):
        self.k_list = sorted(k) if isinstance(k, list) else [k]
        self.voxel = voxel if voxel is not None else 1
        self.compute_density, self.compute_occlusion = density, occlusion
        self.verbose = verbose
        assert density or occlusion, "At least one of `density` or `occlusion` must be True."

    def __call__(self, pos, images: SameSettingImageData, device='cuda', neighbors=None):
        """pos [N,3] (row i = point i of `images.mappings`); returns `images` with the new columns
        appended to `images.mappings.features` (on the mappings' device)."""
        from ..._lib import launch
        assert images.mappings is not None
        maps = images.mappings
        in_device = maps.pointers.device
        dev = torch.device(device)
        xyz = pos.float().to(dev).contiguous()
        n = xyz.shape[0]
        assert n == maps.num_groups, "one position per point of the mappings is expected"
        kmax = self.k_list[-1]
        if neighbors is None:
            neighbors = knn_grid(xyz, kmax)
        neighbors = neighbors.to(dev).long().contiguous()
        vptr = maps.pointers.to(dev).contiguous()
        img = maps.images.to(dev).long().contiguous()
        view_point = torch.arange(n, device=dev).repeat_interleave(vptr[1:] - vptr[:-1])
        V, nk = img.shape[0], len(self.k_list)
        width = nk * (int(self.compute_density) + int(self.compute_occlusion))
        out = torch.empty((V, width), dtype=torch.float32, device=dev)
        klist = torch.tensor(self.k_list, dtype=torch.int32, device=dev)
        launch("dva_neighborhood_features", dev, xyz, neighbors, kmax, vptr, img, view_point, klist, nk,
               float(self.voxel), int(self.compute_density), int(self.compute_occlusion), out, n, V)
        out = out.to(in_device)
        maps.features = out if not maps.has_features else torch.cat([maps.features, out], dim=1)
        return images
