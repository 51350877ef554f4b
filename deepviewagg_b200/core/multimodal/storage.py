"""Flat on-disk format for point-image mappings (SURVEY §8(f) rank 4).

The reference pickles `(data_list, image_data_list)` tuples with `torch.save`
(datasets/segmentation/multimodal/s3dis.py:541-603): loading a sample unpickles nested
CSRData objects and then indexes them in Python.  Here one file holds the arrays of the
two-level CSR exactly as the kernels consume them (SURVEY Appendix B):

    magic "DVAMAP01" | u64 header bytes | JSON header | 64-byte aligned raw little-endian arrays

    per setting s:  s{s}/pointers   int64 [N+1]     view CSR over points
                    s{s}/images     int64 [V]       image of each view
                    s{s}/atomic_ptr int64 [V+1]     pixel CSR over views
                    s{s}/pixels     int16|int32 [P,2]
                    s{s}/features   float32 [V,F]   (optional)
                    s{s}/pos, s{s}/opk float64 [B,3] and any per-image extras
                    s{s}/x          [B,C,H,W] feature maps, raw bytes in their memory layout
                                    (channels-last maps stored as [B,H,W,C]) (optional)
                    s{s}/mask       bool [W_proj,H_proj] projection mask (optional)

    image paths, when set, are kept in the JSON header.

Arrays are read back through `numpy.memmap` (no copy, no unpickling) and uploaded with one
pinned, asynchronous H2D copy each; `load_image_data(..., device='cuda')` therefore costs one
`cudaMemcpyAsync` per array.  A file written from an ImageData reloads to identical tensors.
"""
import json
import struct

import numpy as np
import torch

from .image import ImageData, ImageMapping, SameSettingImageData
from .csr import CSRData

MAGIC = b"DVAMAP01"
_ALIGN = 64


def _np(t):
    return t.detach().cpu().contiguous().numpy()


def save_image_data(path, image_data):
    """Write an ImageData (or one SameSettingImageData) to `path`."""
    settings = list(image_data) if isinstance(image_data, ImageData) else [image_data]
    arrays, meta = {}, {"settings": []}
    for s, im in enumerate(settings):
        m = im.mappings
        assert m is not None, "settings without mappings cannot be stored"
        pre = f"s{s}/"
        arrays[pre + "pointers"] = _np(m.pointers)
        arrays[pre + "images"] = _np(m.images)
        arrays[pre + "atomic_ptr"] = _np(m.values[1].pointers)
        arrays[pre + "pixels"] = _np(m.pixels)
        if m.has_features:
            arrays[pre + "features"] = _np(m.features)
        for key in ("pos", "opk", "crop_offsets"):
            if getattr(im, key) is not None:
                arrays[pre + key] = _np(getattr(im, key))
        for key, val in im.extras.items():
            if isinstance(val, torch.Tensor):
                arrays[pre + "extras/" + key] = _np(val)
        st = dict(ref_size=list(im.ref_size), proj_upscale=im.proj_upscale, downscale=im.downscale,
                  crop_size=list(im.crop_size), num_views=int(im.num_views), has_features=bool(m.has_features))
        if im.x is not None:
            cl = (not im.x.is_contiguous()) and im.x.is_contiguous(memory_format=torch.channels_last)
            arrays[pre + "x"] = _np(im.x.permute(0, 2, 3, 1) if cl else im.x)
            st["x_channels_last"] = bool(cl)
        if im.mask is not None:
            arrays[pre + "mask"] = _np(im.mask)
        if im.path is not None:
            st["path"] = [str(p) for p in im.path]
        meta["settings"].append(st)
    offset, table = 0, {}
    for name, a in arrays.items():
        offset = (offset + _ALIGN - 1) // _ALIGN * _ALIGN
        table[name] = dict(dtype=a.dtype.str, shape=list(a.shape), offset=offset)
        offset += a.nbytes
    meta["arrays"] = table
    header = json.dumps(meta).encode()
    base = (len(MAGIC) + 8 + len(header) + _ALIGN - 1) // _ALIGN * _ALIGN
    with open(path, "wb") as f:
        f.write(MAGIC)
        f.write(struct.pack("<Q", len(header)))
        f.write(header)
        for name, a in arrays.items():
            f.seek(base + table[name]["offset"])
            f.write(a.astype(a.dtype.newbyteorder("<"), copy=False).tobytes())
        f.truncate(max(f.tell(), base + offset))
    return path


def read_header(path):
    with open(path, "rb") as f:
        if f.read(len(MAGIC)) != MAGIC:
            raise ValueError(f"{path}: not a DVAMAP01 file")
        (n,) = struct.unpack("<Q", f.read(8))
        meta = json.loads(f.read(n).decode())
    base = (len(MAGIC) + 8 + n + _ALIGN - 1) // _ALIGN * _ALIGN
    return meta, base


def _tensor(path, base, entry, device, pin):
    shape = tuple(entry["shape"])
    count = int(np.prod(shape)) if shape else 1
    if count == 0:
        return torch.empty(shape, dtype=getattr(torch, np.dtype(entry["dtype"]).name)).to(device)
    mm = np.memmap(path, dtype=np.dtype(entry["dtype"]), mode="r", offset=base + entry["offset"], shape=shape)
    dev = torch.device(device)
    if dev.type == "cpu":
        return torch.from_numpy(np.array(mm))      # private, writable copy
    host = torch.empty(shape, dtype=getattr(torch, mm.dtype.name), pin_memory=pin)
    host.numpy()[...] = mm                       # page cache -> pinned staging, one pass
    return host.to(dev, non_blocking=pin)


def load_image_data(path, device="cpu", pin=True):
    """Read a file written by save_image_data back into an ImageData on `device`."""
    meta, base = read_header(path)
    t = lambda name: _tensor(path, base, meta["arrays"][name], device, pin)  # noqa: E731
    out = []
    for s, st in enumerate(meta["settings"]):
        pre = f"s{s}/"
        names = [n for n in meta["arrays"] if n.startswith(pre)]
        atomic = CSRData(t(pre + "atomic_ptr"), t(pre + "pixels"), dense=False)
        values = [t(pre + "images"), atomic]
        flags = [True, False]
        if st["has_features"]:
            values.append(t(pre + "features"))
            flags.append(False)
        maps = ImageMapping(t(pre + "pointers"), *values, dense=False, is_index_value=flags)
        extras = {n[len(pre + "extras/"):]: t(n) for n in names if n.startswith(pre + "extras/")}
        opt = lambda key: t(pre + key) if pre + key in meta["arrays"] else None  # noqa: E731
        im = SameSettingImageData(pos=opt("pos"), opk=opt("opk"), ref_size=tuple(st["ref_size"]),
                                  proj_upscale=st["proj_upscale"], downscale=st["downscale"],
                                  crop_size=tuple(st["crop_size"]), crop_offsets=opt("crop_offsets"),
                                  num_views=st["num_views"], **extras)
        im.mappings = maps
        if pre + "x" in meta["arrays"]:
            x = t(pre + "x")
            im._x = x.permute(0, 3, 1, 2) if st.get("x_channels_last") else x
        if pre + "mask" in meta["arrays"]:
            im.mask = t(pre + "mask")
        if "path" in st:
            im.path = np.array(st["path"], dtype=object)
        out.append(im)
    return ImageData(out)
