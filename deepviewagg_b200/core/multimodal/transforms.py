"""Per-sample image transforms with the reference's names, arguments and defaults
(torch_points3d/core/data_transform/multimodal/image.py), for the chain every shipped dataset config runs
between loading a sample and the forward pass, and the two that open every config's pre_transform chain
(LoadImages -> NonStaticMask -> MapImages -> NeighborhoodBasedMappingFeatures):

  LoadImages -> NonStaticMask
  ToImageData -> SelectMappingFromPointId -> CenterRoll -> PickImagesFromMappingArea -> CropImageGroups
    -> PickImagesFromMemoryCredit -> JitterMappingFeatures -> ColorJitter -> RandomHorizontalFlip
    -> ToFloatImage -> Normalize

Every transform is called as `data, images = T(data, images)`.  `data` is duck-typed: the mapping key is an
attribute (`data.mapping_index`) and the point count is `data.num_nodes` or `data.pos.shape[0]`, so a PyG
`Data` and a `types.SimpleNamespace` both work.  Containers on CUDA run the kernels of
csrc/image_transforms.cu and csrc/image_color.cu (no fallback); containers on the CPU (data-loader workers) run
a torch restatement of the same arithmetic.  Both give the reference's result bit for bit, including its random
draws: the draws are made on the CPU generators (torch and numpy) exactly as the reference makes them.  The one
exception is ColorJitter's contrast mean, which is exact here (see ColorJitter).

Each docstring lists the host synchronisations of the CUDA path.  Intrinsics are not adjusted and `rollings`
are not persisted by storage.py.  The colour transforms keep the memory format of `images.x`.
"""
import copy

import numpy as np
import torch

from ... import ops
from .image import ImageData, SameSettingImageData, _expand

MAPPING_KEY = 'mapping_index'


def _num_nodes(data):
    n = getattr(data, 'num_nodes', None)
    return int(n) if n is not None else int(data.pos.shape[0])


def _clone(data):
    return data.clone() if hasattr(data, 'clone') else copy.copy(data)


def _pixel_image_ids(mappings):
    return _expand(mappings.images, mappings.values[1].pointers)


def _image_stats(images, ref_w=None):
    """(count [n] int64, bbox [n, 4] (x_min, x_max, y_min, y_max), occupancy [n, 256] bool or [n, 8] int32
    bitmaps) of the current mappings; empty images get count 0 and bbox 0 (torch_scatter's empty -> 0)."""
    m, n = images.mappings, images.num_views
    if m.pointers.is_cuda:
        return ops.mapping_image_stats(m.images, m.values[1].pointers, m.pixels, n, ref_w=ref_w)
    idx = _pixel_image_ids(m)
    count = torch.bincount(idx, minlength=n)[:n]
    pix = m.pixels.long()
    i2 = idx.view(-1, 1).expand(-1, 2)
    big = torch.iinfo(torch.long).max
    mn = torch.full((n, 2), big, dtype=torch.long).scatter_reduce(0, i2, pix, 'amin')
    mx = torch.full((n, 2), -big, dtype=torch.long).scatter_reduce(0, i2, pix, 'amax')
    bbox = torch.stack((mn[:, 0], mx[:, 0], mn[:, 1], mx[:, 1]), dim=1)
    bbox[count == 0] = 0
    occ = None
    if ref_w is not None:
        q = (pix[:, 0].float() * 256 / ref_w).long() & 255             # image.py:1005, then .byte()
        occ = torch.zeros((n, 256), dtype=torch.bool)
        occ[idx, q] = True
    return count, bbox, occ


class ImageTransform:
    """Dispatch of the reference (image.py:29-57): lists are mapped item by item; an `ImageData` is
    processed setting by setting unless the transform sets `_PROCESS_IMAGE_DATA`, in which case a
    `SameSettingImageData` is wrapped into an `ImageData` first.

    Deliberate difference: a transform that turns one setting into several (CropImageGroups) returns one
    flat `ImageData` on an `ImageData` input, where the reference would nest `ImageData` in `ImageData`."""

    _PROCESS_IMAGE_DATA = False

    def _process(self, data, images):
        raise NotImplementedError

    def __call__(self, data, images):
        if isinstance(data, list):
            assert isinstance(images, list) and len(data) == len(images), \
                "List(Data) items and List(SameSettingImageData) must have the same lengths."
            out = [self.__call__(da, im) for da, im in zip(data, images)]
            data_out, images_out = [list(x) for x in zip(*out)]
        elif isinstance(images, ImageData) and not self._PROCESS_IMAGE_DATA:
            out = [self.__call__(_clone(data), im) for im in images]
            flat = []
            for _, im in out:
                flat.extend(list(im) if isinstance(im, ImageData) else [im])
            images_out = ImageData(flat)
            data_out = out[0][0] if len(out) > 0 else data
        else:
            if isinstance(images, SameSettingImageData) and self._PROCESS_IMAGE_DATA:
                images = ImageData([images])
            data_out, images_out = self._process(data, images)
        return data_out, images_out

    def __repr__(self):
        attr_repr = ', '.join([f'{k}={v}' for k, v in self.__dict__.items()])
        return f'{self.__class__.__name__}({attr_repr})'


def _set_ref_size(images, ref_size):
    """image.py:492-505: a new ref_size resets crop_size."""
    images.ref_size = tuple(ref_size)
    images.crop_size = images.ref_size


class LoadImages(ImageTransform):
    """Load the images of `images.path` into `images.x` (image.py:69-102): the given ref_size, crop_size,
    crop_offsets and downscale are set on the container first, then SameSettingImageData.load reads the images
    wrt that state.  Syncs: none on the device; the host decodes every image."""

    def __init__(self, ref_size=None, crop_size=None, crop_offsets=None, downscale=None, show_progress=False):
        self.ref_size = ref_size
        self.crop_size = crop_size
        self.crop_offsets = crop_offsets
        self.downscale = downscale
        self.show_progress = show_progress

    def _process(self, data, images):
        if self.ref_size is not None:
            _set_ref_size(images, self.ref_size)
        if self.crop_size is not None:
            images.crop_size = tuple(self.crop_size)
        if self.crop_offsets is not None:
            images.crop_offsets = self.crop_offsets
        if self.downscale is not None:
            images._downscale = self.downscale
        if self.show_progress:
            print("    LoadImages...")
        images.load(show_progress=self.show_progress)
        return data, images


class NonStaticMask(ImageTransform):
    """Projection mask of the pixels that are not identical across images (image.py:105-159), e.g. to drop
    the camera rig or the vehicle body: `n_sample` images drawn with the reference's
    torch.multinomial(torch.arange(n, dtype=torch.float), n_sample) on the CPU generator are read at
    proj_size, and a pixel is True when every channel of some drawn image differs from the first drawn one.
    With fewer than 2 images the mask is all True.  Image 0 has weight 0 in that draw, so it is drawn only
    after every other image (reproduced as is).  CUDA: read_images + dva_nonstatic_mask; syncs: none on the
    device."""

    def __init__(self, ref_size=None, proj_upscale=None, n_sample=5):
        self.ref_size = tuple(ref_size) if ref_size is not None else None
        self.proj_upscale = proj_upscale
        self.n_sample = n_sample

    def _process(self, data, images):
        if self.ref_size is not None:
            _set_ref_size(images, self.ref_size)
        if self.proj_upscale is not None:
            images.proj_upscale = self.proj_upscale
        n_sample = min(self.n_sample, images.num_views)
        if n_sample < 2:
            mask = torch.ones(images.proj_size, dtype=torch.bool)
        else:
            idx = torch.multinomial(torch.arange(images.num_views, dtype=torch.float), n_sample)
            imgs = images.read_images(idx=idx, size=images.proj_size)
            if imgs.is_cuda:
                mask = ops.nonstatic_mask(imgs)
            else:
                mask = (imgs[1:] != imgs[:1]).all(dim=1).any(dim=0).t().contiguous()
        images.mask = mask
        return data, images


class SelectMappingFromPointId(ImageTransform):
    """Keep the mappings of the points `data.mapping_index` (in that order) and the images they see, then
    renumber `data.mapping_index` to arange(num_nodes) (image.py:615-644).  Syncs: those of
    SameSettingImageData.select_points."""

    def __init__(self):
        self.key = MAPPING_KEY

    def _process(self, data, images):
        assert hasattr(data, self.key)
        assert isinstance(images, SameSettingImageData)
        assert images.mappings is not None
        images = images.select_points(getattr(data, self.key), mode='pick')
        setattr(data, self.key, torch.arange(_num_nodes(data), device=images.device))
        return data, images


class CenterRoll(ImageTransform):
    """Roll equirectangular images and mappings along the width so that each image's mappings sit as close
    to the image centre as possible (image.py:962-1037): the quantised widths are rolled by every candidate
    of range(0, 256, 256 // angular_res) and the first roll of least span + centre distance wins.
    CUDA: dva_mapping_image_stats (occupancy) -> dva_center_roll -> update_rollings.  Syncs: one, to check
    that every image has a mapping."""

    def __init__(self, angular_res=16):
        assert isinstance(angular_res, int)
        assert angular_res <= 256
        self.angular_res = angular_res

    def _process(self, data, images):
        msg = f"{self.__class__.__name__} cannot operate if images and mappings underwent prior cropping or resizing."
        assert images.mappings is not None, "No mappings found in images."
        assert images.ref_size[0] == images.img_size[0], msg
        assert images.crop_size is None or images.crop_size[0] == images.ref_size[0], msg
        assert images.downscale is None or images.downscale == 1, msg
        if images.mappings.images.shape[0] == 0:
            return data, images
        ref_w = images.ref_size[0]
        count, _, occ = _image_stats(images, ref_w=ref_w)
        if occ.is_cuda:
            rollings = ops.center_roll(occ, self.angular_res, ref_w)
        else:
            rolls = torch.arange(0, 256, int(256 / self.angular_res)).byte()
            w = (torch.arange(256).view(1, -1) + rolls.long().view(-1, 1)) & 255             # [R, 256]
            on = occ.unsqueeze(1)                                                           # [n, 1, 256]
            w_min = torch.where(on, w, 256).amin(dim=2)
            w_max = torch.where(on, w, -1).amax(dim=2)
            empty = w_max < 0
            w_min[empty], w_max[empty] = 0, 0
            w_cost = (w_max - w_min).int() + ((w_max.float() + w_min) / 2. - 128).abs().int()
            roll_idx = (w_cost == w_cost.amin(dim=1, keepdim=True)).int().argmax(dim=1)    # first argmin
            rollings = (rolls[roll_idx] / 256. * ref_w).long()
        assert bool((count > 0).all()), "Image indices discrepancy in the rollings."
        images.update_rollings(rollings)
        return data, images


class PickImagesFromMappingArea(ImageTransform):
    """Keep the images whose mapping area (pixel count, or bounding-box area with use_bbox) exceeds
    area_ratio of the image, largest first, at most n_max (image.py:713-762).  The comparison is in fp32;
    equal areas keep the higher image index first (stable ascending sort, then flip).  Syncs: the boolean
    selection, then those of SameSettingImageData.__getitem__."""

    def __init__(self, area_ratio=0.02, n_max=None, n_min=0, use_bbox=False):
        self.area_ratio = area_ratio
        self.n_max = n_max if n_max is not None and n_max >= 1 else None
        self.n_min = n_min if n_max is not None and n_min >= 0 else 0
        self.use_bbox = use_bbox

    def _process(self, data, images):
        assert images.mappings is not None, "No mappings found in images."
        threshold = images.img_size[0] * images.img_size[1] * self.area_ratio
        count, bbox, _ = _image_stats(images)
        if not self.use_bbox:
            areas = count.float()
        else:
            bbox = bbox.int()
            areas = (bbox[:, 1] - bbox[:, 0]) * (bbox[:, 3] - bbox[:, 2])
        n_max = images.num_views if self.n_max is None else self.n_max
        idx = torch.sort(areas, stable=True).indices.flip(0)
        idx = idx[areas[idx].float() > threshold][:n_max]
        # the reference's fallback slices an empty index, so it stays empty (kept as is)
        if idx.shape[0] == 0 and images.num_views > 0 and self.n_min > 0:
            idx = idx[:self.n_min]
        return data, images[idx]


class CropImageGroups(ImageTransform):
    """Distribute the images over crop sizes (min_size, min_size), then doubling width and height in turn
    up to img_size, by the padded bounding box of their mappings, and crop each group with its boxes
    centred and clamped to the image (image.py:1040-1141).  Returns an ImageData with one setting per crop
    size, in the order the sizes were first used.  CUDA: dva_mapping_image_stats, the family loop on the
    host, one dva_image_remap per family.  Syncs: one bounding-box read (4 integers per image), then those
    of SameSettingImageData.__getitem__ and ImageMapping.crop per family."""

    def __init__(self, padding=0, min_size=64):
        assert padding >= 0, f"Expected a positive scalar but got {padding} instead."
        assert ((min_size & (min_size - 1)) == 0) & (min_size != 0), \
            f"Expected a power of two but got {min_size} instead."
        self.padding = padding
        self.min_size = min_size

    def _process(self, data, images):
        assert images.mappings is not None, "No mappings found in images."
        if images.num_views == 0:
            return data, ImageData([images])
        _, bbox, _ = _image_stats(images)
        bbox = bbox.cpu().long()
        w_min, w_max, h_min, h_max = bbox.unbind(1)
        img_size = tuple(images.img_size)
        w_min = torch.clamp(w_min - self.padding, 0)
        h_min = torch.clamp(h_min - self.padding, 0)
        w_max = torch.clamp(w_max + self.padding, 0, img_size[0])
        h_max = torch.clamp(h_max + self.padding, 0, img_size[1])
        widths = w_max - w_min
        heights = h_max - h_min

        crop_families = {}
        size = (self.min_size, self.min_size)
        i_crop = 0
        image_ids = torch.arange(images.num_views)
        while all(a <= b for a, b in zip(size, img_size)):
            if image_ids.shape[0] == 0:
                break
            if size == img_size:
                crop_families[size] = image_ids
                break
            valid_ids = torch.logical_and(widths[image_ids] <= size[0], heights[image_ids] <= size[1])
            if image_ids[valid_ids].shape[0] > 0:
                crop_families[size] = image_ids[valid_ids]
            image_ids = image_ids[~valid_ids]
            size = (min(size[0] * 2 ** ((i_crop + 1) % 2), img_size[0]),
                    min(size[1] * 2 ** (i_crop % 2), img_size[1]))
            i_crop += 1
        if img_size not in crop_families.keys() and image_ids.shape[0] > 0:
            crop_families[img_size] = image_ids

        for size, idx in crop_families.items():
            # centre the box in the crop, fp32 / 2., truncation, clamp (image.py:1129-1135)
            off_x = torch.clamp((w_min[idx] - (size[0] - widths[idx]) / 2.).long(), 0, img_size[0] - size[0])
            off_y = torch.clamp((h_min[idx] - (size[1] - heights[idx]) / 2.).long(), 0, img_size[1] - size[1])
            offsets = torch.stack((off_x, off_y), dim=1).long()
            crop_families[size] = images[idx].update_cropping(size, offsets)
        return data, ImageData(list(crop_families.values()))


class _CoverageIndexCPU:
    """CPU restatement of ops.CoverageIndex: unseen[g] starts at g's view count; pick(g) marks g's points
    seen and takes every newly seen point off the count of each image that sees it."""

    def __init__(self, gimg, vpoint, n_img, num_points):
        self.gimg, self.vpoint, self.n_img = gimg, vpoint, n_img
        self.by_img = torch.sort(gimg, stable=True).indices
        self.img_off = torch.cat([torch.zeros(1, dtype=torch.long), torch.bincount(gimg, minlength=n_img).cumsum(0)])
        self.by_pt = torch.sort(vpoint, stable=True).indices
        self.pt_off = torch.cat([torch.zeros(1, dtype=torch.long),
                                 torch.bincount(vpoint, minlength=num_points).cumsum(0)])
        self.unseen = (self.img_off[1:] - self.img_off[:-1]).int()
        self.seen = torch.zeros(num_points, dtype=torch.bool)

    def pick(self, g):
        pts = self.vpoint[self.by_img[self.img_off[g]:self.img_off[g + 1]]]
        new = pts[~self.seen[pts]]
        self.seen[new] = True
        cnt = self.pt_off[new + 1] - self.pt_off[new]
        start = torch.repeat_interleave(self.pt_off[new], cnt)
        within = torch.arange(int(cnt.sum())) - torch.repeat_interleave(cnt.cumsum(0) - cnt, cnt)
        views = self.by_pt[start + within]
        self.unseen -= torch.bincount(self.gimg[views], minlength=self.n_img).int()


class PickImagesFromMemoryCredit(ImageTransform):
    """Pick images of all settings at random until a pixel credit is spent, weighting each by its size
    and, with k_coverage > 0, by how many not-yet-seen points it carries (image.py:765-874).  The loop
    runs on the host with the reference's numpy float64 arithmetic and one np.random.choice per pick, so a
    given np.random seed gives the reference's picks; each setting keeps its images in pick order.
    CUDA with k_coverage > 0: the unseen counts come from dva_coverage_index / dva_coverage_pick, with one
    sync per pick (a copy of n_img int32 to pinned memory).  With k_coverage = 0 there is no device work
    and no sync besides those of SameSettingImageData.__getitem__."""

    _PROCESS_IMAGE_DATA = True

    def __init__(self, credit=None, img_size=[], k_coverage=0, n_img=0):
        if credit is not None:
            self.credit = credit
        elif len(img_size) == 2 and n_img > 0:
            self.credit = img_size[0] * img_size[1] * n_img
        else:
            raise ValueError("Either credit or img_size and n_img must be provided.")
        self.use_coverage = k_coverage > 0
        self.k_coverage = k_coverage

    def _coverage_index(self, data, images):
        gimg, vpoint, base = [], [], 0
        N = max([_num_nodes(data)] + [im.num_points for im in images])
        for im in images:
            m = im.mappings
            gimg.append(m.images + base)
            vpoint.append(_expand(torch.arange(m.num_groups, device=m.device), m.pointers))
            base += im.num_views
        gimg, vpoint = torch.cat(gimg), torch.cat(vpoint)
        if gimg.is_cuda:
            return ops.CoverageIndex(gimg, vpoint, base, N)
        return _CoverageIndexCPU(gimg, vpoint, base, N)

    def _process(self, data, images):
        if images.num_views == 0:
            return data, images
        picked = [[] for _ in range(images.num_views)]
        img_indices = [[i, j] for i, im in enumerate(images) for j in range(im.num_views)]
        gids = list(range(len(img_indices)))
        img_sizes = [images[i].img_size[0] * images[i].img_size[1] for i, j in img_indices]
        if self.use_coverage:
            cov = self._coverage_index(data, images)
            host = torch.empty(cov.unseen.shape, dtype=torch.int32, pin_memory=cov.unseen.is_cuda)

        credit = self.credit
        assert credit > 0 and credit >= min(img_sizes), \
            f"Insufficient credit={credit} to pick any of the provided images with min_size={min(img_sizes)}."
        while credit > 0 and len(img_indices) > 0 and credit >= min(img_sizes):
            for idx in range(len(img_indices), 0, -1):
                if img_sizes[idx - 1] > credit:
                    img_indices.pop(idx - 1)
                    img_sizes.pop(idx - 1)
                    gids.pop(idx - 1)
            if self.use_coverage:
                if cov.unseen.is_cuda:
                    host.copy_(cov.unseen, non_blocking=True)
                    torch.cuda.current_stream(cov.unseen.device).synchronize()
                else:
                    host.copy_(cov.unseen)
                unseen = host.numpy()
                w_cov = np.array([int(unseen[g]) for g in gids])
                w_cov = self.k_coverage * w_cov / (w_cov.max() + 1)
            else:
                w_cov = np.zeros(len(img_indices))
            w_size = np.array(img_sizes) / np.array(img_sizes).max()
            weights = w_size + w_cov
            probas = weights / weights.sum()
            idx = np.random.choice(np.arange(probas.shape[0]), p=probas)
            i, j = img_indices.pop(idx)
            s = img_sizes.pop(idx)
            g = gids.pop(idx)
            picked[i].append(j)
            credit -= s
            if self.use_coverage:
                cov.pick(g)
        images = ImageData([im[torch.LongTensor(idx)] for im, idx in zip(images, picked) if len(idx) > 0])
        return data, images


class JitterMappingFeatures(ImageTransform):
    """Add sigma * N(0, 1) noise clamped to [-clip, clip] to the mapping features (image.py:934-959).  The
    noise is drawn on the CPU default generator exactly as the reference draws it and then moved, so the
    result is the reference's under torch.manual_seed whatever the device.  Syncs: none (one host to
    device copy)."""

    def __init__(self, sigma=0.02, clip=0.03):
        self.sigma = sigma
        self.clip = clip

    def _process(self, data, images):
        if images.mappings is None or not images.mappings.has_features:
            return data, images
        noise = self.sigma * torch.randn(images.mappings.features.shape)
        noise = noise.clamp(-self.clip, self.clip)
        m = images.mappings.clone()
        m.features = m.features + noise.to(m.device)
        images.mappings = m
        return data, images


class RandomHorizontalFlip(ImageTransform):
    """With probability p (torch.rand(1) <= p on the CPU generator), flip `x` along the width and set the
    mapping pixels to width - 1 - x (image.py:1195-1218).  CUDA: one dva_image_remap copy.  Syncs: none."""

    def __init__(self, p=0.50):
        self.p = p

    def _process(self, data, images):
        assert images.x is not None, "RandomHorizontalFlip needs loaded images (x)."
        if torch.rand(1) <= self.p:
            if images.x.is_cuda:
                images.x = ops.image_remap(images.x, flip=True)
            else:
                images.x = images.x[..., torch.arange(images.x.shape[-1] - 1, -1, -1)]
            width = images.x.shape[-1]
            if images.mappings is not None:
                m = images.mappings.clone()
                m.values[1] = m.values[1].clone()
                pix = m.pixels.clone()
                pix[:, 0] = width - 1 - pix[:, 0]
                m.pixels = pix
                images.mappings = m
        return data, images


class ToImageData(ImageTransform):
    """Wrap a SameSettingImageData into ImageData([images]) (image.py:64-68).  An ImageData input comes back as
    the same settings in one flat ImageData."""

    def _process(self, data, images):
        return data, ImageData([images])


def _jitter_range(value, name):
    """torchvision ColorJitter._check_input for a scalar: [max(0, 1 - v), 1 + v], None (no draw, no op) when v == 0"""
    if value < 0:
        raise ValueError(f"If {name} is a single number, it must be non negative.")
    lo, hi = max(1.0 - float(value), 0.0), 1.0 + float(value)
    return None if lo == hi == 1.0 else (lo, hi)


def _gray_u8(x):
    """torchvision rgb_to_grayscale on [B, 3, H, W] uint8: (0.2989 r + 0.587 g) + 0.114 b in fp32, truncated"""
    r, g, b = x.unbind(dim=-3)
    return (0.2989 * r + 0.587 * g + 0.114 * b).to(torch.uint8).unsqueeze(-3)


def _blend_u8(img, other, ratio):
    """torchvision _blend for uint8: fp32(ratio) * img + fp32(1 - ratio) * other, clamped to [0, 255], truncated"""
    return (ratio * img + (1.0 - ratio) * other).clamp(0, 255).to(torch.uint8)


def color_jitter_torch(x, ops_seq):
    """torch restatement of dva_color_jitter_u8 (the CPU path; on CUDA tensors the multi-pass chain a user would
    write): the ops of `ops_seq` ((name, factor) in the drawn order) on a [B, 3, H, W] uint8 tensor, with the
    exact contrast mean fp32(float64(S) / float64(H W)) of the integer grayscale sum S.  Keeps x's memory format."""
    fmt = ops._memory_format(x)
    HW = x.shape[-1] * x.shape[-2]
    for name, f in ops_seq:
        if name == "brightness":
            x = _blend_u8(x, torch.zeros_like(x), f)
        elif name == "saturation":
            x = _blend_u8(x, _gray_u8(x), f)
        else:
            s = _gray_u8(x).sum(dim=(1, 2, 3), dtype=torch.int64).double()
            mean = (s / torch.full_like(s, float(HW))).float().view(-1, 1, 1, 1)      # true division on any device
            x = _blend_u8(x, mean, f)
    return x.contiguous(memory_format=fmt)


class ColorJitter(ImageTransform):
    """Randomly change the brightness, contrast and saturation of `images.x` (image.py:1249-1259), restating
    torchvision's ColorJitter without depending on it.  Ranges are [max(0, 1 - v), 1 + v] (off when v == 0);
    the draw is torchvision's get_params on the CPU default generator: torch.randperm(4), then one
    uniform_(lo, hi) each for brightness, contrast and saturation, in that order, for the ones that are on.  The
    ops run in the drawn order with torchvision's uint8 arithmetic (fp32 blends truncated to uint8 after every
    op).  Each setting of an ImageData gets its own draw; a setting without images consumes its draw too.

    `images.x` must be [B, 3, H, W] uint8 (ColorJitter comes before ToFloatImage in every config).  One
    deliberate difference: the contrast mean is float32(float64(S) / float64(H W)) of the exact integer sum S of
    the grayscale bytes, where torchvision's fp32 torch.mean depends on the reduction order and may be an ulp
    away; a pixel can then differ by 1 where its blend value lies within that shift of an integer.
    CUDA: dva_color_jitter_u8 (one pass, or two with contrast).  Syncs: none."""

    def __init__(self, brightness=0, contrast=0, saturation=0):
        self.brightness = brightness
        self.contrast = contrast
        self.saturation = saturation
        self._ranges = (_jitter_range(brightness, "brightness"), _jitter_range(contrast, "contrast"),
                        _jitter_range(saturation, "saturation"))

    def get_params(self):
        """(fn_idx [4] int64, [(name, factor) of the active ops in the drawn order])"""
        fn_idx = torch.randperm(4)
        factors = [None if r is None else float(torch.empty(1).uniform_(r[0], r[1])) for r in self._ranges]
        names = ("brightness", "contrast", "saturation")
        return fn_idx, [(names[i], factors[i]) for i in fn_idx.tolist() if i < 3 and factors[i] is not None]

    def _process(self, data, images):
        x = images.x
        if x is None or x.dim() != 4 or x.shape[1] != 3 or x.dtype != torch.uint8:
            got = None if x is None else (tuple(x.shape), x.dtype)
            raise TypeError(f"ColorJitter expects images.x as a [B, 3, H, W] uint8 tensor, got {got}")
        _, seq = self.get_params()
        if x.shape[0] == 0 or len(seq) == 0:
            return data, images
        images.x = ops.color_jitter_u8(x, seq) if x.is_cuda else color_jitter_torch(x, seq)
        return data, images

    def __repr__(self):
        return (f"{self.__class__.__name__}(brightness={self.brightness}, contrast={self.contrast}, "
                f"saturation={self.saturation})")


class ToFloatImage(ImageTransform):
    """[0, 255] uint8 images to [0, 1] fp32: x.float() / 255 with true division, as on the CPU
    (image.py:1221-1232); loads the images first when `x` is None.  CUDA: dva_image_to_float, for uint8 or
    fp32 `x` (a CUDA division by a Python scalar would multiply by the reciprocal).  Syncs: none."""

    def _process(self, data, images):
        if images.x is None:
            images.load()
        x = images.x
        if x.is_cuda:
            images.x = ops.image_to_float(x)
        else:
            images.x = (x.float() / 255).contiguous(memory_format=ops._memory_format(x))
        return data, images


class Normalize(ImageTransform):
    """(x - mean_c) / std_c with true division (image.py:1271-1282): torchvision's normalize, sub_(mean).div_(std)
    with [C, 1, 1] tensors of x's dtype.  Non-float `x` raises a TypeError, as in torchvision.  CUDA:
    dva_image_to_float with the statistics passed by value, fp32 `x` with 1 to 4 channels.  Syncs: none."""

    def __init__(self, mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225]):
        self.mean = mean
        self.std = std

    def _process(self, data, images):
        x = images.x
        if x is None or not torch.is_floating_point(x):
            raise TypeError(f"Input tensor should be a float tensor. Got {None if x is None else x.dtype}.")
        if x.is_cuda and x.dtype != torch.float32:
            raise TypeError(f"Normalize on CUDA runs on float32 images, got {x.dtype}")
        std = torch.as_tensor(self.std, dtype=x.dtype)
        if (std == 0).any():
            raise ValueError(f"std evaluated to zero after conversion to {x.dtype}, leading to division by zero.")
        if x.is_cuda:
            images.x = ops.image_to_float(x, self.mean, self.std)
        else:
            mean = torch.as_tensor(self.mean, dtype=x.dtype).view(-1, 1, 1)
            images.x = ((x - mean) / std.view(-1, 1, 1)).contiguous(memory_format=ops._memory_format(x))
        return data, images
