"""Point <-> image <-> pixel mapping containers with the reference's interface
(torch_points3d/core/multimodal/image.py), restricted to what the view-aggregation path touches:

  ImageMapping / ImageMappingBatch       image.py:1707-2347   two-level CSR (point -> view -> pixel)
  SameSettingImageData / ...Batch        image.py:177-1407    feature maps + mappings of one setting
  ImageData / ImageBatch                 image.py:1409-1704   list of settings; view_cat_* indexing
  sparse_interpolation                   image.py:105-170

Integer layout is the reference's bit for bit (Appendix B of SURVEY.md): pointers int64, images
int64 [V], atomic CSR pointers int64 [V+1] over pixels intK [P,2] (x, y), features f32 [V,F],
is_index_value = [True, False(, False)].  Sorting is stable (utils/multimodal.py), so results
equal the reference up to the order of equal keys.  Intrinsics bookkeeping and plotting are out of scope
(dataset side).  Rolling and cropping of loaded samples (update_rollings / update_cropping, used by
core/multimodal/transforms.py) are kept, and so is image loading (read_images / load, image.py:973-1101):
Pillow on CPU containers, the Pillow-exact resize kernel of csrc/image_resample.cu on CUDA containers.
"""
import copy
from typing import List

import numpy as np
import torch

from ... import _lib, ops
from ...utils.multimodal import composite_key, lexargsort, lexargunique, lexunique, tensor_idx
from .csr import CSRBatch, CSRData, pointers_from_sorted

_PIX_CODES = {torch.int16: 0, torch.int32: 1, torch.int64: 2}


def _native_mapping_build(point_ids, image_ids, pixels, features, num_points, feat_row=None, feat_on=None,
                          dedupe=False):
    """dva_mapping_build on CUDA tensors: bucket the items by point (counting sort), order every
    point's items with a warp rank sort on (image[, x, y], source index), cut views / dedupe pixels,
    average the view features -- all on the current stream, ONE device->host read (the output sizes).
    Returns an ImageMapping."""
    dev = point_ids.device
    n = int(point_ids.shape[0])
    if pixels.dtype not in _PIX_CODES:
        pixels = pixels.long()
    pixels = pixels.contiguous()
    point_ids, image_ids = point_ids.long().contiguous(), image_ids.long().contiguous()
    F = 0 if features is None else int(features.shape[1])
    if F > 16:
        raise NotImplementedError("mapping features wider than 16 columns")
    feat = features.float().contiguous() if features is not None else None
    view_ptr = torch.empty(num_points + 1, dtype=torch.long, device=dev)
    images_out = torch.empty(n, dtype=torch.long, device=dev)
    atomic_ptr = torch.empty(n + 1, dtype=torch.long, device=dev)
    pixels_out = torch.empty_like(pixels)
    feat_out = torch.empty((n, F), dtype=torch.float32, device=dev) if feat is not None else None
    counts = torch.empty(3, dtype=torch.long, device=dev)
    ws = _lib.workspace(_lib.load().dva_mapping_build_workspace_bytes(n, num_points), dev)
    if feat_on is not None:
        feat_on = feat_on.to(torch.uint8).contiguous()
    if feat_row is not None:
        feat_row = feat_row.long().contiguous()
    _lib.launch("dva_mapping_build", dev, point_ids, image_ids, pixels, _PIX_CODES[pixels.dtype], feat, feat_row,
                feat_on, F, n, int(num_points), int(bool(dedupe)), view_ptr, images_out, atomic_ptr, pixels_out,
                feat_out, None, counts, ws, ws.numel())
    V, P, status = counts.tolist()                           # the only synchronisation
    if status != 0:
        raise IndexError("from_dense: point ids outside [0, num_points)")
    atomic = CSRData(atomic_ptr[:V + 1], pixels_out[:P], dense=False)
    if feat is None:
        return ImageMapping(view_ptr, images_out[:V], atomic, dense=False, is_index_value=[True, False])
    return ImageMapping(view_ptr, images_out[:V], atomic, feat_out[:V].to(features.dtype), dense=False,
                        is_index_value=[True, False, False])


# ------------------------------------------------------------------------------------------------
# segment helpers usable on either device (containers may be built on the dataloader's CPU side)
# ------------------------------------------------------------------------------------------------
def _segment_mean(src, pointers):
    if src.is_cuda:
        return ops.segment_csr(src, pointers, reduce='mean')
    counts = (pointers[1:] - pointers[:-1])
    dense = torch.arange(counts.numel()).repeat_interleave(counts)
    out = torch.zeros((counts.numel(),) + tuple(src.shape[1:]), dtype=src.dtype).index_add_(0, dense, src)
    return out / counts.clamp(min=1).to(src.dtype).view(-1, *([1] * (src.dim() - 1)))


def _counts(pointers):
    return pointers[1:] - pointers[:-1]


def _expand(values, pointers):
    """values[i] repeated count_i times."""
    return values.repeat_interleave(_counts(pointers), dim=0)


def sparse_interpolation(features, coords, batch, padding_mode='border'):
    """Bilinear interpolation of [B,C,H,W] maps at per-row float coordinates in [0,1]
    (image.py:105-170): pad 1 px, p = coords * (h, w) + 0.5, corners floor(p) / floor(p + 1),
    weight of a corner = |prod(p - opposite corner)|."""
    assert features.dim() == 4 and coords.shape[0] == batch.shape[0] and coords.shape[1] == 2
    pad = {'zeros': torch.nn.ZeroPad2d, 'border': torch.nn.ReplicationPad2d,
           'reflection': torch.nn.ReflectionPad2d}
    if padding_mode not in pad:
        raise NotImplementedError(f"Unknown padding_mode='{padding_mode}'")
    padded = pad[padding_mode](1)(features)
    h, w = features.shape[2:]
    pix = coords * torch.tensor([[h, w]], dtype=coords.dtype, device=features.device) + 0.5
    top, bottom = torch.floor(pix[:, 0]), torch.floor(pix[:, 0] + 1)
    left, right = torch.floor(pix[:, 1]), torch.floor(pix[:, 1] + 1)
    out = 0
    for (r, c), (ro, co) in (((top, left), (bottom, right)), ((top, right), (bottom, left)),
                             ((bottom, left), (top, right)), ((bottom, right), (top, left))):
        wgt = ((pix[:, 0] - ro) * (pix[:, 1] - co)).abs().unsqueeze(1)
        out = out + wgt * padded[batch, :, r.long(), c.long()]
    return out


# ------------------------------------------------------------------------------------------------
# ImageMapping
# ------------------------------------------------------------------------------------------------
class ImageMapping(CSRData):
    """CSRData format for point-image-pixel mappings (image.py:1707-2343)."""

    @staticmethod
    def from_dense(point_ids, image_ids, pixels, features, num_points=None):
        """image.py:1728-1795: sort by (point, image); atomic CSR over (point, image) runs;
        per-view feature = mean over its pixels; view CSR over points; empty points inserted."""
        assert point_ids.ndim == 1 and point_ids.shape == image_ids.shape
        assert point_ids.shape[0] == pixels.shape[0]
        assert features is None or point_ids.shape[0] == features.shape[0]
        if point_ids.is_cuda and num_points is not None and (features is None or features.shape[1] <= 16):
            # native builder: no sort over all items, no intermediate tensors, one host read
            return _native_mapping_build(point_ids, image_ids, pixels, features, int(num_points))
        order = lexargsort(point_ids, image_ids)
        image_ids, point_ids, pixels = image_ids[order], point_ids[order], pixels[order]
        if features is not None:
            features = features[order]
        key, _ = composite_key(point_ids, image_ids)
        atomic = CSRData(key, pixels, dense=True)
        last = atomic.pointers[1:] - 1
        image_ids, point_ids = image_ids[last], point_ids[last]
        if features is not None:
            features = _segment_mean(features, atomic.pointers)
        n_seen = int(point_ids.max().item()) + 1 if point_ids.numel() else 0
        num_points = n_seen if num_points is None else max(int(num_points), n_seen)
        pointers = pointers_from_sorted(point_ids, num_points)
        if features is None:
            return ImageMapping(pointers, image_ids, atomic, dense=False, is_index_value=[True, False])
        return ImageMapping(pointers, image_ids, atomic, features, dense=False,
                            is_index_value=[True, False, False])

    def is_cuda_native(self):
        """True when the native re-indexing kernels apply (CUDA tensors, <= 16 feature columns, pixel
        coordinates that fit the 16-bit sort key)."""
        return (self.pointers.is_cuda and (not self.has_features or self.features.shape[1] <= 16)
                and self.pixels.dtype in (torch.int16, torch.int32, torch.int64))

    def debug(self):
        super().debug()
        assert len(self.values) == 2 or self.has_features
        assert isinstance(self.values[1], CSRData) and len(self.values[1].values) == 1

    @property
    def points(self):
        return torch.arange(self.num_groups, device=self.device)

    @property
    def images(self):
        return self.values[0]

    @images.setter
    def images(self, images):
        self.values[0] = images.to(self.device)

    @property
    def has_features(self):
        return len(self.values) == 3

    @property
    def features(self):
        return self.values[2] if self.has_features else None

    @features.setter
    def features(self, features):
        if self.has_features:
            if features is None:
                self.values.pop(-1)
                self.is_index_value = self.is_index_value[:2]
            else:
                self.values[2] = features.to(self.device)
        elif features is not None:
            self.values.append(features.to(self.device))
            self.is_index_value = torch.tensor([True, False, False])

    @property
    def pixels(self):
        return self.values[1].values[0]

    @pixels.setter
    def pixels(self, pixels):
        self.values[1].values[0] = pixels.to(self.device)

    @staticmethod
    def get_batch_type():
        return ImageMappingBatch

    @property
    def bounding_boxes(self):
        """(w_min, w_max, h_min, h_max) per image (image.py:1859-1869)."""
        image_ids = _expand(self.images, self.values[1].pointers)
        n = int(image_ids.max().item()) + 1 if image_ids.numel() else 0
        pix = self.pixels.long()
        idx = image_ids.view(-1, 1).expand(-1, 2)
        big = torch.iinfo(torch.long).max
        mn = torch.full((n, 2), big, dtype=torch.long, device=self.device).scatter_reduce(0, idx, pix, 'amin')
        mx = torch.full((n, 2), -big, dtype=torch.long, device=self.device).scatter_reduce(0, idx, pix, 'amax')
        return mn[:, 0], mx[:, 0], mn[:, 1], mx[:, 1]

    @property
    def feature_map_indexing(self):
        """Index tuple into [B,C,H,W] maps: (image per pixel, ..., y, x) (image.py:1871-1885)."""
        idx_batch = _expand(self.images, self.values[1].pointers)
        return (idx_batch.long(), ..., self.pixels[:, 1].long(), self.pixels[:, 0].long())

    @property
    def atomic_csr_indexing(self):
        return self.values[1].pointers

    @property
    def view_csr_indexing(self):
        return self.pointers

    def rescale_images(self, ratio):
        return self.downscale_images(1 / ratio) if ratio < 1 else self.upscale_images(ratio)

    def downscale_images(self, ratio):
        """Pixel coordinates at a `ratio` times coarser resolution: pix // ratio (image.py:1916-1980).

        NB the reference keys its duplicate removal on the per-pixel item ids (`lexargunique(ids,
        pix_x, pix_y)`, image.py:1944-1959), which are all distinct: nothing is ever removed and the
        atomic pointers are unchanged -- pixels of a view that collapse onto one coarse pixel stay
        duplicated (harmless for the max atomic pool).  Reproduced as is."""
        assert ratio >= 1, f"Invalid image subsampling ratio: {ratio}. Must be larger than 1."
        out = self.clone()
        if ratio == 1:
            return out
        atomic = out.values[1].clone()
        pix = atomic.values[0]
        atomic.values[0] = torch.stack(((pix[:, 0] // ratio).long(), (pix[:, 1] // ratio).long()),
                                       dim=1).to(pix.dtype)
        out.values[1] = atomic
        return out

    def upscale_images(self, ratio, center=True):
        """image.py:1982-2027."""
        assert ratio >= 1, f"Invalid image upsampling ratio: {ratio}. Must be larger than 1."
        out = self.clone()
        if ratio == 1:
            return out
        out.values[1] = out.values[1].clone()
        pix = out.values[1].values[0]
        shift = ratio / 2 if center else 0
        out.values[1].values[0] = (pix.float() * ratio + shift).long().to(pix.dtype)
        return out

    def _view_point_ids(self):
        return _expand(torch.arange(self.num_groups, device=self.device), self.pointers)

    def _from_views(self, keep, values):
        """New mapping over the same points from a subset of views (rows `keep`, in view order)."""
        point_ids = self._view_point_ids()[keep]
        pointers = pointers_from_sorted(point_ids, self.num_groups)
        return self.__class__(pointers, *values, dense=False, is_index_value=self.is_index_value)

    def select_images(self, idx):
        """Keep the mappings to images in idx and renumber them idx[i] -> i (image.py:2029-2093)."""
        idx = tensor_idx(idx).to(self.device)
        assert idx.unique().numel() == idx.shape[0], "Index must not contain duplicates."
        if self.num_items == 0:
            return self.clone()
        if idx.shape[0] == 0:
            values = [v[torch.zeros(0, dtype=torch.long, device=self.device)] for v in self.values]
            return self.__class__(torch.zeros_like(self.pointers), *values, dense=False,
                                  is_index_value=self.is_index_value)
        lut = torch.full((max(int(idx.max().item()), int(self.images.max().item())) + 1,), -1,
                         dtype=torch.long, device=self.device)
        lut[idx] = torch.arange(idx.shape[0], device=self.device)
        new_img = lut[self.images]
        keep = torch.where(new_img >= 0)[0]
        values = [v[keep] for v in self.values]
        values[0] = new_img[keep]
        return self._from_views(keep, values)

    def select_views(self, view_mask):
        """image.py:2095-2165 -> (mapping, selected image indices or None)."""
        if isinstance(view_mask, np.ndarray):
            view_mask = torch.from_numpy(view_mask)
        assert view_mask.dtype == torch.bool and view_mask.dim() == 1 and view_mask.shape[0] == self.num_items
        if self.num_items == 0:
            return self.clone()
        keep = torch.where(view_mask.to(self.device))[0]
        values = [v[keep] for v in self.values]
        if keep.numel() == 0:
            out = self.__class__(torch.zeros_like(self.pointers), *values, dense=False,
                                 is_index_value=self.is_index_value)
            return out, torch.zeros(0, dtype=torch.long)
        img_idx = values[0].unique()
        if img_idx.numel() < int(self.images.max().item()) + 1:
            lut = torch.full((int(img_idx.max().item()) + 1,), -1, dtype=torch.long, device=self.device)
            lut[img_idx] = torch.arange(img_idx.shape[0], device=self.device)
            values[0] = lut[values[0]]
        else:
            img_idx = None
        return self._from_views(keep, values), img_idx

    def select_points(self, idx, mode='pick'):
        """'pick': self[idx]; 'merge': points i -> idx[i] are agglomerated, duplicate
        (point', image, pixel) mappings removed, features averaged per (point', image)
        (image.py:2167-2277).  'merge' runs after every strided 3D convolution (modules.py:232-234)."""
        assert mode in ('pick', 'merge'), f"Unknown mode '{mode}'. Supported modes are ['pick', 'merge']."
        idx = tensor_idx(idx).to(self.device)
        if idx.shape[0] == 0 or self.num_groups == 0:
            return self.clone()
        if self.num_items == 0:
            out = self.clone()
            out.pointers = torch.zeros(idx.shape[0] + 1, dtype=torch.long, device=self.device)
            return out
        if mode == 'pick':
            return self[idx]
        if not idx.shape[0] == self.num_groups > 0:
            return self.clone()
        n_out = int(idx.max().item()) + 1
        if self.is_cuda_native():
            present = torch.zeros(n_out, dtype=torch.bool, device=self.device)
            present[idx] = True
            if not bool(present.all()):              # every output voxel must appear (image.py:2220)
                return self.clone()
            # native path: items = pixels, bucketed by the merged point; a merged view's feature is the mean
            # over its SOURCE VIEWS (image.py:2233-2247), i.e. over the first pixel of every source view
            ap = self.values[1].pointers
            V, P = self.num_items, int(self.pixels.shape[0])
            view_points = idx.repeat_interleave(_counts(self.pointers), output_size=V)
            pcount = _counts(ap)
            view_of_pixel = torch.arange(V, device=self.device).repeat_interleave(pcount, output_size=P)
            first = torch.zeros(P, dtype=torch.uint8, device=self.device)
            first[ap[:-1][pcount > 0]] = 1
            return _native_mapping_build(view_points[view_of_pixel], self.images[view_of_pixel], self.pixels,
                                         self.features if self.has_features else None, n_out,
                                         feat_row=view_of_pixel, feat_on=first, dedupe=True)
        if idx.unique().numel() != n_out:
            return self.clone()
        view_points = _expand(idx, self.pointers)
        features = self.features
        if self.has_features and self.num_items > 1:
            # mean feature per merged (point', image) view, redistributed to its source views
            key, _ = composite_key(view_points, self.images)
            uniq, inv = torch.unique(key, return_inverse=True)
            sums = torch.zeros((uniq.numel(), features.shape[1]), dtype=features.dtype,
                               device=self.device).index_add_(0, inv, features)
            cnt = torch.zeros(uniq.numel(), dtype=features.dtype, device=self.device).index_add_(
                0, inv, torch.ones_like(inv, dtype=features.dtype))
            features = (sums / cnt.view(-1, 1))[inv]
        ap = self.values[1].pointers
        point_ids = _expand(view_points, ap)
        image_ids = _expand(self.images, ap)
        if features is not None:
            features = _expand(features, ap)
        pixels = self.pixels
        keep = lexargunique(point_ids, image_ids, pixels[:, 0], pixels[:, 1])
        return ImageMapping.from_dense(point_ids[keep], image_ids[keep], pixels[keep],
                                       features[keep] if features is not None else None, num_points=n_out)

    def crop(self, crop_size, crop_offsets):
        """image.py:2279-2342."""
        ap = self.values[1].pointers
        image_ids = _expand(self.images, ap)
        pixels = self.pixels - crop_offsets.to(self.device)[image_ids]     # promotes to the offsets' dtype (int64), like image.py:2302
        size = torch.tensor(crop_size, device=self.device)
        inside = torch.where((pixels >= 0).all(dim=1) & (pixels < size).all(dim=1))[0]
        if inside.shape[0] == 0:
            out = self.clone()
            out.values[1] = out.values[1].clone()
            out.pixels = pixels
            return out
        point_ids = _expand(self._view_point_ids(), ap)
        features = _expand(self.features, ap) if self.has_features else None
        return ImageMapping.from_dense(point_ids[inside], image_ids[inside], pixels[inside],
                                       features[inside] if features is not None else None,
                                       num_points=self.num_groups)


class ImageMappingBatch(ImageMapping, CSRBatch):
    """Batch wrapper for ImageMapping (image.py:2345-2347)."""
    __csr_type__ = ImageMapping


# ------------------------------------------------------------------------------------------------
# SameSettingImageData
# ------------------------------------------------------------------------------------------------
class SameSettingImageData:
    """Feature maps `x` [B,C,H,W] of B images sharing one acquisition setting + their mappings
    (image.py:177-1287).  Only the state the aggregation path reads is kept: pose arrays are carried
    opaquely in `extras` (same per-image leading dimension) so that image selection stays consistent.
    `path` [B] (numpy object array) names the image files read by read_images / load; `mask` [W_proj, H_proj]
    bool is the projection mask MapImages applies (a shared setting: kept by indexing, clone and to, taken
    from the first item when batching, and not part of settings_hash, as in the reference)."""

    # decoded native-resolution bytes staged per chunk by the CUDA read_images (S3DIS panoramas are 25 MB each)
    _READ_CHUNK_BYTES = 256 << 20

    def __init__(self, pos=None, opk=None, ref_size=(512, 256), proj_upscale=2, downscale=1, crop_size=None,
                 crop_offsets=None, x=None, mappings=None, num_views=None, rollings=None, path=None, mask=None,
                 **extras):
        self.path = np.array(path, dtype=object).reshape(-1) if path is not None else None
        self.pos = pos.double() if pos is not None else None
        self.opk = opk.double() if opk is not None else None
        self._num_views = num_views
        self.ref_size = tuple(ref_size)
        self.proj_upscale = proj_upscale
        self.crop_size = tuple(crop_size) if crop_size is not None else self.ref_size
        self.crop_offsets = crop_offsets
        self._downscale = downscale
        self.extras = {k: v for k, v in extras.items() if v is not None}
        self._x = None
        self._mappings = None
        self.x = x
        self.mappings = mappings
        # per-image width rolling wrt ref_size (image.py:553-576); not part of settings_hash (_shared_keys)
        self.rollings = rollings if rollings is not None else \
            torch.zeros(self.num_views, dtype=torch.long, device=self.device)
        self._mask = None
        self.mask = mask

    # -- sizes
    @property
    def num_views(self):
        if self.pos is not None:
            return self.pos.shape[0]
        if self._num_views is not None:
            return self._num_views
        if self._x is not None:
            return self._x.shape[0]
        return len(self.path) if self.path is not None else 0

    @property
    def num_points(self):
        return self.mappings.num_groups if self.mappings is not None else 0

    @property
    def img_size(self):
        return tuple(int(v / self.downscale) for v in self.crop_size)

    @property
    def mapping_size(self):
        return self.crop_size

    @property
    def downscale(self):
        return self._downscale

    @property
    def proj_size(self):
        """Size (W, H) of the projection map and of the mask: ref_size * proj_upscale (image.py:543-551)."""
        return tuple(int(v * self.proj_upscale) for v in self.ref_size)

    @property
    def mask(self):
        """Projection mask: None or a [W_proj, H_proj] bool tensor (image.py:952-971)."""
        return self._mask

    @mask.setter
    def mask(self, mask):
        if mask is None:
            self._mask = None
            return
        assert mask.dtype == torch.bool, f"Expected a dtype=torch.bool but got dtype={mask.dtype} instead."
        assert tuple(mask.shape) == self.proj_size, \
            f"Expected mask of size {self.proj_size} but got {tuple(mask.shape)} instead."
        self._mask = mask.to(self.device)

    @property
    def pixel_dtype(self):
        for dtype in (torch.int16, torch.int32, torch.int64):
            if torch.iinfo(dtype).max >= max(self.ref_size):
                return dtype

    # -- features and mappings
    @property
    def x(self):
        return self._x

    @x.setter
    def x(self, x):
        """Setting features at a new resolution updates `downscale` (image.py:756-787)."""
        if x is None:
            self._x = None
            return
        assert isinstance(x, torch.Tensor) and x.shape[0] == self.num_views, \
            f"Expected a tensor of shape ({self.num_views}, :, H, W) but got {tuple(x.shape)} instead."
        scale = max(self.img_size[0] / x.shape[3], self.img_size[1] / x.shape[2])
        self._downscale = self.downscale * scale
        self._x = x

    @property
    def mappings(self):
        return self._mappings

    @mappings.setter
    def mappings(self, mappings):
        assert mappings is None or isinstance(mappings, ImageMapping)
        self._mappings = mappings

    @property
    def device(self):
        for t in (self._x, self.pos, self._mappings.pointers if self._mappings is not None else None):
            if t is not None:
                return t.device
        return torch.device('cpu')

    @property
    def settings_hash(self):
        return hash((self.ref_size, self.proj_upscale, self.downscale, self.crop_size))

    @staticmethod
    def get_batch_type():
        return SameSettingImageBatch

    def __len__(self):
        return self.num_views

    def clone(self):
        out = copy.copy(self)
        out.extras = dict(self.extras)
        out._x = self._x.clone() if self._x is not None else None
        out._mappings = self._mappings.clone() if self._mappings is not None else None
        out.rollings = self.rollings.clone()
        return out

    def to(self, device):
        out = copy.copy(self)
        mv = lambda t: t.to(device) if isinstance(t, torch.Tensor) else t  # noqa: E731
        out.pos, out.opk, out.crop_offsets = mv(self.pos), mv(self.opk), mv(self.crop_offsets)
        out.rollings = mv(self.rollings)
        out.extras = {k: mv(v) for k, v in self.extras.items()}
        out._x = mv(self._x)
        out._mappings = self._mappings.to(device) if self._mappings is not None else None
        out._mask = mv(self._mask)
        return out

    def __getitem__(self, idx):
        """Select images (no duplicates); mappings follow (image.py:1109-1148)."""
        idx = tensor_idx(idx).to(self.device)
        assert idx.unique().numel() == idx.shape[0], "Index must not contain duplicates."
        sel = lambda t: t[idx.to(t.device)] if isinstance(t, torch.Tensor) else t  # noqa: E731
        out = copy.copy(self)
        out.pos, out.opk, out.crop_offsets = sel(self.pos), sel(self.opk), sel(self.crop_offsets)
        out.rollings = sel(self.rollings)
        out.extras = {k: sel(v) for k, v in self.extras.items()}
        out._num_views = int(idx.shape[0])
        out._x = self._x[idx] if self._x is not None else None
        out._mappings = self._mappings.select_images(idx) if self._mappings is not None else None
        out.path = self.path[idx.cpu().numpy()] if self.path is not None else None
        out._mask = self._mask.clone() if self._mask is not None else None
        return out

    def select_points(self, idx, mode='pick'):
        """image.py:826-907: 'pick' also drops the images no selected point sees."""
        idx = tensor_idx(idx).to(self.device)
        if self.mappings is None or idx.shape[0] == 0:
            return self.clone()
        if len(self) == 0:
            return self.clone()
        if mode == 'pick':
            mappings = self.mappings.select_points(idx, mode=mode)
            seen = lexunique(mappings.images) if mappings.num_items > 0 else []
            self_mappings, self._mappings = self._mappings, None
            images = self[seen]
            self._mappings = self_mappings
            images.mappings = mappings.select_images(seen)
            return images
        if mode == 'merge':
            images = self.clone()
            if not idx.shape[0] == self.num_points > 0:
                return images
            if idx.unique().numel() != int(idx.max().item()) + 1:
                return images
            images.mappings = images.mappings.select_points(idx, mode=mode)
            return images
        raise ValueError(f"Unknown point selection mode '{mode}'.")

    # -- rolling and cropping (image.py:578-628, 688-720)
    def update_rollings(self, rollings):
        """Roll `x` and the mappings along the width by `rollings` [B] int64, wrt ref_size: torch.roll
        semantics, x[..., j] <- x[..., (j - r) mod W], and pixel x -> (x + r) % ref_W in pixel_dtype.  Images
        are taken as circular along the width; prior cropping or resizing is refused, as in the reference.
        CUDA containers roll `x` with one dva_image_remap copy.  No synchronisation."""
        assert self.ref_size[0] == self.img_size[0], \
            "CenterRoll cannot operate if images and mappings underwent prior cropping or resizing."
        assert self.crop_size is None or self.crop_size == self.ref_size, \
            "CenterRoll cannot operate if images and mappings underwent prior cropping or resizing."
        assert self.downscale is None or self.downscale == 1, \
            "CenterRoll cannot operate if images and mappings underwent prior cropping or resizing."
        self.rollings = rollings
        if self.x is not None:
            if self.x.is_cuda:
                self.x = ops.image_remap(self.x, rolls=self.rollings.to(self.x.device))
            else:
                self.x = torch.stack([torch.roll(im, int(r), dims=-1) for im, r in zip(self.x, self.rollings.cpu())])
        if self.mappings is not None:
            m = self.mappings.clone()
            m.values[1] = m.values[1].clone()
            pix = m.pixels.clone()
            pix_roll = _expand(self.rollings.to(m.device)[m.images], m.values[1].pointers)
            pix[:, 0] = ((pix[:, 0].long() + pix_roll) % self.ref_size[0]).to(self.pixel_dtype)
            m.pixels = pix
            self.mappings = m
        return self

    def update_cropping(self, crop_size, crop_offsets):
        """Crop `x` and the mappings to `crop_size` (W, H) at per-image `crop_offsets` [B, 2] (x, y), both
        wrt the current img_size.  The stored crop_size and crop_offsets are wrt ref_size: scaled by
        `downscale` and accumulated over successive crops (a crop_offsets of None counts as zeros).  The
        mappings go through ImageMapping.crop; CUDA containers crop `x` with one dva_image_remap copy.
        Camera intrinsics are not adjusted: intrinsics bookkeeping belongs to the dataset side.  No
        synchronisation."""
        crop_offsets = crop_offsets.long()
        base = self.crop_offsets if self.crop_offsets is not None else \
            torch.zeros((self.num_views, 2), dtype=torch.long, device=self.device)
        self.crop_size = tuple(int(v * self.downscale) for v in crop_size)
        self.crop_offsets = (base + crop_offsets.to(base.device) * self.downscale).long()
        if self.x is not None:
            if self.x.is_cuda:
                self.x = ops.image_remap(self.x, (crop_size[1], crop_size[0]), offsets=crop_offsets.to(self.x.device))
            else:
                self.x = torch.stack([im[:, o[1]:o[1] + crop_size[1], o[0]:o[0] + crop_size[0]]
                                      for im, o in zip(self.x, crop_offsets.tolist())])
        if self.mappings is not None:
            self.mappings = self.mappings.crop(crop_size, crop_offsets)
        return self

    # -- image loading (image.py:973-1101)
    def load(self, show_progress=False):
        """Read the images of `path` into `x` at ref_size with the container's rollings, crop_size, crop_offsets
        and downscale (image.py:973-989), on the container's device.  See read_images."""
        crop_offsets = self.crop_offsets if self.crop_offsets is not None else \
            torch.zeros((self.num_views, 2), dtype=torch.long)
        self._x = self.read_images(size=self.ref_size, rollings=self.rollings, crop_size=self.crop_size,
                                   crop_offsets=crop_offsets, downscale=self.downscale,
                                   show_progress=show_progress).to(self.device)
        return self

    def read_images(self, idx=None, size=None, rollings=None, crop_size=None, crop_offsets=None, downscale=None,
                    show_progress=False):
        """Read the images `path[idx]` as a [B, 3, H, W] uint8 tensor in channels-last memory, as the reference
        does (image.py:991-1101): decode to RGB, resize to `size` (W, H) with Pillow's default BICUBIC filter,
        roll every image sideways by `rollings` (out[:, x] = in[:, (x + r) mod W], i.e. torch.roll by -r, the
        opposite of update_rollings), then crop `crop_size` at `crop_offsets` or, when `downscale` is set,
        resize that box to int(crop_size / downscale).  A crop box must lie inside the resized image.

        CPU containers run Pillow.  CUDA containers decode on the host and stage runs of consecutive images of
        one native size (at most _READ_CHUNK_BYTES decoded) in pinned memory, copy them asynchronously and
        resize / roll / crop them with ops.image_resample and ops.image_remap, bit for bit what Pillow gives.
        Host work: decoding; no device->host read."""
        if idx is None:
            idx = np.arange(self.num_views)
        elif isinstance(idx, int):
            idx = np.array([idx])
        elif isinstance(idx, torch.Tensor):
            idx = np.asarray(idx.cpu())
        elif isinstance(idx, slice):
            idx = np.arange(self.num_views)[idx]
        idx = np.asarray(idx).reshape(-1)
        assert self.path is not None and len(self.path) == self.num_views, \
            "read_images needs one path per image in 'path'."
        size = tuple(int(v) for v in (size if size is not None else self.img_size))
        if rollings is not None:
            assert rollings.dtype == torch.int64, f"Expected dtype=torch.int64 but got dtype={rollings.dtype} instead."
            assert rollings.shape[0] == idx.shape[0], \
                f"Expected tensor of shape {idx.shape[0]} but got {rollings.shape[0]} instead."
        else:
            rollings = torch.zeros(idx.shape[0], dtype=torch.long)
        assert bool(crop_size) == bool(crop_offsets is not None), \
            "If either 'crop_size' or 'crop_offsets' is specified, both must be specified."
        if crop_size is not None:
            crop_size = tuple(int(v) for v in crop_size)
            assert len(crop_size) == 2, f"Expected len(crop_size)=2 but got {len(crop_size)} instead."
            assert all(a <= b for a, b in zip(crop_size, size)), \
                f"Expected crop_size to be smaller than size but got size={size} and crop_size={crop_size} instead."
            assert crop_offsets.dtype == torch.int64, \
                f"Expected dtype=torch.int64 but got dtype={crop_offsets.dtype} instead."
            assert tuple(crop_offsets.shape) == (idx.shape[0], 2), \
                f"Expected tensor of shape {(idx.shape[0], 2)} but got {tuple(crop_offsets.shape)} instead."
        else:
            crop_size = size
            crop_offsets = torch.zeros((idx.shape[0], 2), dtype=torch.long)
        if downscale is not None:
            assert downscale >= 1, f"Expected scalar larger than 1 but got {downscale} instead."
        offsets = crop_offsets.cpu().long()
        assert bool((offsets >= 0).all()) and bool((offsets + torch.tensor(crop_size) <= torch.tensor(size)).all()), \
            f"Crop boxes of size {crop_size} must lie inside the {size} images."
        paths = self.path[idx]
        if show_progress:
            from tqdm.auto import tqdm
            paths = tqdm(paths)
        end_size = crop_size if downscale is None else tuple(int(v / downscale) for v in crop_size)
        from PIL import Image
        if self.device.type == 'cuda':
            return _read_images_cuda(list(paths), size, rollings.cpu().long(), crop_size, offsets, downscale,
                                     end_size, self.device, self._READ_CHUNK_BYTES)
        w, h = crop_size
        arrays = []
        for p, r, (left, top) in zip(paths, rollings.cpu().tolist(), offsets.tolist()):
            im = Image.open(p).convert('RGB').resize(size)
            if r % size[0]:
                im = Image.fromarray(np.roll(np.asarray(im), -(r % size[0]), axis=1))
            box = (left, top, left + w, top + h)
            im = im.crop(box) if downscale is None else im.resize(end_size, box=box)
            arrays.append(np.asarray(im))
        return torch.from_numpy(np.stack(arrays)).permute(0, 3, 1, 2)

    # -- indexing for the pools
    @property
    def feature_map_indexing(self):
        return self.mappings.feature_map_indexing if self.mappings is not None else None

    @property
    def atomic_csr_indexing(self):
        return self.mappings.atomic_csr_indexing if self.mappings is not None else None

    @property
    def view_csr_indexing(self):
        return self.mappings.view_csr_indexing if self.mappings is not None else None

    @property
    def mapping_features(self):
        return self.mappings.features

    def scaled_mappings(self, interpolate=False):
        """Mappings at the resolution of `x` (image.py:1271-1275): re-deduplicated pixel CSR unless
        interpolating."""
        return self.mappings if interpolate else self.mappings.rescale_images(1 / self.downscale)

    def get_mapped_features(self, interpolate=False):
        """[P, C] features of the mapped pixels (image.py:1262-1287)."""
        scale = 1 / self.downscale
        mappings = self.scaled_mappings(interpolate)
        if interpolate and scale != 1:
            if self.x.is_cuda:   # bilinear corners read straight from the map, no padded copy
                from ... import ops
                return ops.sparse_interpolation_pixels(self.x, mappings.feature_map_indexing[0],
                                                       mappings.pixels, self.mapping_size)
            resolution = torch.tensor([self.mapping_size], dtype=torch.float, device=self.device)
            coords = (mappings.pixels / (resolution - 1))[:, [1, 0]]
            return sparse_interpolation(self.x, coords, mappings.feature_map_indexing[0])
        return self.x[mappings.feature_map_indexing]

    def __repr__(self):
        return (f"{self.__class__.__name__}(num_views={self.num_views}, num_points={self.num_points}, "
                f"device={self.device})")


def _read_images_cuda(paths, size, rollings, crop_size, offsets, downscale, end_size, device, chunk_bytes):
    """CUDA body of SameSettingImageData.read_images: [B, 3, H, W] uint8, channels-last, on `device`."""
    from PIL import Image
    n = len(paths)
    native = [Image.open(p).size for p in paths]            # header only, no decoding
    out = torch.empty((n, end_size[1], end_size[0], 3), dtype=torch.uint8, device=device)
    w, h = crop_size
    rolls = -(rollings % size[0])
    boxes = torch.cat([offsets, offsets + torch.tensor([[w, h]])], dim=1)
    i = 0
    while i < n:
        W0, H0 = native[i]
        j = i + 1
        while j < n and native[j] == (W0, H0) and (j + 1 - i) * W0 * H0 * 3 <= chunk_bytes:
            j += 1
        staged = torch.empty((j - i, H0, W0, 3), dtype=torch.uint8, pin_memory=True)
        for k in range(i, j):
            staged[k - i].numpy()[...] = np.asarray(Image.open(paths[k]).convert('RGB'))
        x = staged.to(device, non_blocking=True).permute(0, 3, 1, 2)
        x = ops.image_resample(x, size)
        r = rolls[i:j]
        if downscale is None:
            x = ops.image_remap(x, (h, w), rolls=ops._pinned_to(r.numpy(), device),
                                offsets=ops._pinned_to(offsets[i:j].numpy(), device))
        else:
            if bool((r != 0).any()):
                x = ops.image_remap(x, rolls=ops._pinned_to(r.numpy(), device))
            x = ops.image_resample(x, end_size, boxes=boxes[i:j].float())
        out[i:j] = x.permute(0, 2, 3, 1)
        i = j
    return out.permute(0, 3, 1, 2)


class SameSettingImageBatch(SameSettingImageData):
    """image.py:1290-1406."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self.__sizes__ = None

    @property
    def num_batch_items(self):
        return len(self.__sizes__) if self.__sizes__ is not None else 0

    @staticmethod
    def from_data_list(items):
        assert isinstance(items, list) and len(items) > 0
        assert all(im.settings_hash == items[0].settings_hash for im in items), \
            "All SameSettingImageData values for shared settings must be the same."
        cat = lambda ts: torch.cat(ts) if all(t is not None for t in ts) else None  # noqa: E731
        first = items[0]
        extras = {k: cat([im.extras.get(k) for im in items]) for k in first.extras}
        mappings = None
        if all(im.mappings is not None for im in items):
            mappings = ImageMappingBatch.from_csr_list([im.mappings for im in items])
        batch = SameSettingImageBatch(
            pos=cat([im.pos for im in items]), opk=cat([im.opk for im in items]), ref_size=first.ref_size,
            proj_upscale=first.proj_upscale, downscale=first.downscale, crop_size=first.crop_size,
            crop_offsets=cat([im.crop_offsets for im in items]), num_views=sum(im.num_views for im in items),
            rollings=cat([im.rollings for im in items]), **extras)
        batch.path = np.concatenate([im.path for im in items]) if all(im.path is not None for im in items) else None
        # the first item's mask serves the batch: masks computed by NonStaticMask may differ slightly
        batch._mask = first.mask
        batch._x = cat([im.x for im in items])
        batch._mappings = mappings
        batch.__sizes__ = np.array([im.num_views for im in items])
        return batch


# ------------------------------------------------------------------------------------------------
# ImageData: list of settings
# ------------------------------------------------------------------------------------------------
class ImageData:
    """Holder for SameSettingImageData items of different settings (image.py:1409-1595)."""

    def __init__(self, image_list: List[SameSettingImageData]):
        self._list = image_list

    @property
    def num_settings(self):
        return len(self)

    @property
    def num_views(self):
        return sum(im.num_views for im in self)

    @property
    def num_points(self):
        return self[0].num_points if len(self) > 0 else 0

    @property
    def x(self):
        return [im.x for im in self]

    @x.setter
    def x(self, x_list):
        assert x_list is None or isinstance(x_list, list)
        if x_list is None or len(x_list) == 0:
            x_list = [None] * self.num_settings
        for im, x in zip(self, x_list):
            im.x = x

    def __len__(self):
        return len(self._list)

    def __getitem__(self, idx):
        if len(self) == 0:
            raise ValueError(f'{self} cannot be indexed because it has length 0.')
        if isinstance(idx, int) and idx < len(self):
            return self._list[idx]
        return self.__class__([self._list[i] for i in tensor_idx(idx).tolist()])

    def __iter__(self):
        for i in range(len(self)):
            yield self[i]

    def select_points(self, idx, mode='pick'):
        return self.__class__([im.select_points(idx, mode=mode) for im in self])

    def clone(self):
        return self.__class__([im.clone() for im in self])

    def to(self, device):
        return self.__class__([im.to(device) for im in self])

    @property
    def device(self):
        return self[0].device if len(self) > 0 else 'cpu'

    @staticmethod
    def get_batch_type():
        return ImageBatch

    def get_mapped_features(self, interpolate=False):
        return [im.get_mapped_features(interpolate=interpolate) for im in self]

    @property
    def feature_map_indexing(self):
        return [im.feature_map_indexing for im in self]

    @property
    def atomic_csr_indexing(self):
        return [im.atomic_csr_indexing for im in self]

    @property
    def view_cat_sorting(self):
        """Permutation that puts the concatenated per-setting views in point order
        (image.py:1549-1574); stable, i.e. ties keep the (setting, view) order."""
        if self.device.type == 'cuda' and self.num_settings > 0:
            return self._view_cat_native()[0]
        dense = torch.cat([
            _expand(torch.arange(im.num_points, device=self.device), im.view_csr_indexing) for im in self])
        return torch.sort(dense, stable=True).indices

    def _view_cat_native(self):
        """(sorting, csr_cat) in closed form (dva_view_cat_sorting): every setting's views are already
        grouped by point, so a view's slot in the merged order is a sum of pointers -- no sort."""
        ptrs = [im.view_csr_indexing.contiguous() for im in self]
        N = int(ptrs[0].numel()) - 1
        sizes = [int(im.mappings.images.shape[0]) if im.mappings is not None else 0 for im in self]
        bases, tot = [], 0
        for sz in sizes:
            bases.append(tot)
            tot += sz
        dev = self.device
        table = torch.tensor([p.data_ptr() for p in ptrs] + bases, dtype=torch.long).to(dev)
        sorting = torch.empty(tot, dtype=torch.long, device=dev)
        csr_cat = torch.empty(N + 1, dtype=torch.long, device=dev)
        _lib.launch("dva_view_cat_sorting", dev, table, table.data_ptr() + 8 * len(ptrs), len(ptrs), N, sorting,
                    csr_cat)
        return sorting, csr_cat

    @property
    def view_cat_csr_indexing(self):
        """Sum of the per-setting view pointers (image.py:1576-1588)."""
        return torch.stack([im.view_csr_indexing for im in self], dim=1).sum(dim=1)

    @property
    def mapping_features(self):
        return [im.mapping_features for im in self]

    def __repr__(self):
        return (f"{self.__class__.__name__}(num_settings={self.num_settings}, num_views={self.num_views}, "
                f"num_points={self.num_points}, device={self.device})")


class ImageBatch(ImageData):
    """Batch of ImageData grouped by setting, with global point re-indexing (image.py:1598-1704)."""

    def __init__(self, image_list):
        super().__init__(image_list)
        self.__il_sizes__ = None
        self.__cum_pts__ = None

    @staticmethod
    def from_data_list(image_data_list):
        assert isinstance(image_data_list, list) and len(image_data_list) > 0
        hashes = []
        for il in image_data_list:
            for im in il:
                if im.settings_hash not in hashes:
                    hashes.append(im.settings_hash)
        n_pts = [il.num_points for il in image_data_list]
        cum = [0]
        for n in n_pts:
            cum.append(cum[-1] + n)
        groups = {h: [] for h in hashes}
        owners = {h: [] for h in hashes}
        for il_idx, il in enumerate(image_data_list):
            for im in il:
                groups[im.settings_hash].append(im)
                owners[im.settings_hash].append(il_idx)
        batches = []
        for h in hashes:
            b = SameSettingImageBatch.from_data_list(groups[h])
            if b.num_points > 0:
                global_idx = torch.cat([torch.arange(cum[i], cum[i + 1]) for i in owners[h]])
                b.mappings.insert_empty_groups(global_idx.to(b.mappings.device), num_groups=cum[-1])
            batches.append(b)
        out = ImageBatch(batches)
        out.__il_sizes__ = [len(il) for il in image_data_list]
        out.__cum_pts__ = torch.tensor(cum)
        return out
