"""Polygon ground-truth masks on the GPU (DESIGN.md f-4): PolygonMasks.crop_and_resize and polygons_to_bitmask /
BitMasks.from_polygon_masks (detectron2/structures/masks.py:22-85, 166-180, 396-420), bit-exact to pycocotools.

The reference rasterizes each proposal's polygons on the host with pycocotools, in a Python loop over proposals, after
copying the boxes to the host.  Here a batch's polygons are packed once (`pack_polygons`, one host-to-device copy per
array) and every proposal or image tile is rasterized by one CTA (csrc/polygon_raster.cuh); mask_head.mask_rcnn_loss takes
the packed batch as `gt_masks` and rasterizes the targets inside its loss kernel.
"""
from typing import List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _C
from ._C import check, ptr, stream_ptr

Tensor = torch.Tensor

__all__ = ["PackedPolygons", "pack_polygons", "polygons_crop_and_resize", "polygons_to_bitmask"]


class PackedPolygons(NamedTuple):
    """A batch's polygons on one device.  coords [V, 2] float64 vertices (x, y); poly_start [P + 1] int32: polygon p is
    vertices [poly_start[p], poly_start[p + 1]); inst_start [G + 1] int32: instance g is polygons [inst_start[g],
    inst_start[g + 1]); image_start (host ints, length images + 1): image i is instances [image_start[i], image_start[i + 1])."""
    coords: Tensor
    poly_start: Tensor
    inst_start: Tensor
    image_start: Tuple[int, ...]

    @property
    def num_instances(self) -> int:
        return self.image_start[-1]


def _as_float64(p) -> np.ndarray:
    if isinstance(p, torch.Tensor):
        p = p.detach().cpu().numpy()
    return np.asarray(p).astype("float64").reshape(-1)


def pack_polygons(polygons_per_image: Sequence[Sequence[Sequence]], device) -> PackedPolygons:
    """polygons_per_image[i] is image i's PolygonMasks.polygons: a list per instance of polygons, each a flat
    [x0, y0, x1, y1, ...] array, list or tensor.  Raises the reference's ValueError for a polygon with an odd number of
    coordinates or fewer than 6 (PolygonMasks.__init__, masks.py:296-309)."""
    flat, poly_start, inst_start, image_start = [], [0], [0], [0]
    for instances in polygons_per_image:
        for polys in instances:
            for p in polys:
                a = _as_float64(p)
                if len(a) % 2 != 0 or len(a) < 6:
                    raise ValueError(f"Cannot create a polygon from {len(a)} coordinates.")
                flat.append(a)
                poly_start.append(poly_start[-1] + len(a) // 2)
            inst_start.append(len(poly_start) - 1)
        image_start.append(len(inst_start) - 1)
    if poly_start[-1] >= 2 ** 31:
        raise ValueError("pack_polygons: more than 2^31 - 1 vertices in one batch")
    coords = np.concatenate(flat) if flat else np.zeros((0,), np.float64)
    dev = torch.device(device)
    return PackedPolygons(torch.from_numpy(coords.reshape(-1, 2)).to(dev),
                          torch.tensor(poly_start, dtype=torch.int32).to(dev),
                          torch.tensor(inst_start, dtype=torch.int32).to(dev), tuple(image_start))


def _batch_args(coords, poly_start, inst_start):
    return (ptr(coords), coords.shape[0], ptr(poly_start), poly_start.shape[0] - 1, ptr(inst_start),
            inst_start.shape[0] - 1)


def _check_packed(coords, poly_start, inst_start):
    _C.require_cuda(coords, poly_start, inst_start)
    if (coords.dtype != torch.float64 or coords.dim() != 2 or coords.shape[1] != 2 or poly_start.dtype != torch.int32
            or inst_start.dtype != torch.int32 or poly_start.dim() != 1 or inst_start.dim() != 1
            or len(poly_start) < 1 or len(inst_start) < 1):
        raise RuntimeError("polygons: expected coords [V, 2] float64, poly_start [P + 1] and inst_start [G + 1] int32")
    return coords.contiguous(), poly_start.contiguous(), inst_start.contiguous()


@torch.library.custom_op("d2b200::polygons_crop_and_resize", mutates_args=(), device_types="cuda")
def _crop_and_resize_op(coords: Tensor, poly_start: Tensor, inst_start: Tensor, boxes: Tensor,
                        mask_index: Optional[Tensor], mask_size: int) -> Tensor:
    coords, poly_start, inst_start = _check_packed(coords, poly_start, inst_start)
    _C.require_cuda(boxes, mask_index)
    if boxes.dim() != 2 or boxes.shape[1] != 4 or (mask_index is not None and mask_index.shape != (boxes.shape[0],)):
        raise RuntimeError("polygons_crop_and_resize: boxes must be K x 4 and mask_index K")
    if not 1 <= mask_size <= _C.POLYGON_MAX_S:
        raise RuntimeError("polygons_crop_and_resize: mask_size must be in [1, %d]" % _C.POLYGON_MAX_S)
    k = boxes.shape[0]
    out = torch.empty((k, mask_size, mask_size), dtype=torch.bool, device=boxes.device)
    if k:
        bx = boxes.to(dtype=torch.float32).contiguous()
        mi = None if mask_index is None else mask_index.to(dtype=torch.int64).contiguous()
        with torch.cuda.device(bx.device):
            check(_C.lib().d2b_polygons_crop_and_resize(*_batch_args(coords, poly_start, inst_start), ptr(bx), ptr(mi), k,
                                                        mask_size, ptr(out), stream_ptr(bx.device)),
                  "polygons_crop_and_resize")
    return out


@_crop_and_resize_op.register_fake
def _(coords, poly_start, inst_start, boxes, mask_index, mask_size):
    return boxes.new_empty((boxes.shape[0], mask_size, mask_size), dtype=torch.bool)


@torch.library.custom_op("d2b200::polygons_to_bitmask", mutates_args=(), device_types="cuda")
def _to_bitmask_op(coords: Tensor, poly_start: Tensor, inst_start: Tensor, height: int, width: int) -> Tensor:
    coords, poly_start, inst_start = _check_packed(coords, poly_start, inst_start)
    if height < 1 or width < 1:
        raise RuntimeError("polygons_to_bitmask: height and width must be positive")
    g = inst_start.shape[0] - 1
    out = torch.empty((g, height, width), dtype=torch.bool, device=coords.device)
    if g:
        with torch.cuda.device(coords.device):
            check(_C.lib().d2b_polygons_to_bitmask(*_batch_args(coords, poly_start, inst_start), height, width, ptr(out),
                                                   stream_ptr(coords.device)), "polygons_to_bitmask")
    return out


@_to_bitmask_op.register_fake
def _(coords, poly_start, inst_start, height, width):
    return coords.new_empty((inst_start.shape[0] - 1, height, width), dtype=torch.bool)


def polygons_crop_and_resize(packed: PackedPolygons, boxes: Tensor, mask_size: int,
                             mask_index: Optional[Tensor] = None) -> Tensor:
    """PolygonMasks.crop_and_resize: boxes [K, 4] (fp32 values; the reference reads them as float32), mask_index [K]
    instance of each box in the packed batch (None: box k <-> instance k, as the reference pairs them).
    Returns [K, mask_size, mask_size] bool on the boxes' device."""
    return _crop_and_resize_op(packed.coords, packed.poly_start, packed.inst_start, boxes, mask_index, int(mask_size))


def polygons_to_bitmask(packed: PackedPolygons, height: int, width: int) -> Tensor:
    """BitMasks.from_polygon_masks(...).tensor of every instance of the packed batch: [G, height, width] bool."""
    return _to_bitmask_op(packed.coords, packed.poly_start, packed.inst_start, int(height), int(width))


def batch_mask_index(packed: PackedPolygons, num_proposals: List[int], mask_index: Optional[List[Tensor]],
                     device) -> Tensor:
    """Per-image ground-truth indices -> indices into the packed batch, on the device and without a host sync: index m of
    image i becomes image_start[i] + m when 0 <= m < that image's instance count, else -1 (so it can never reach another
    image's instance).  mask_index None: proposal k of an image uses that image's instance k."""
    if len(num_proposals) != len(packed.image_start) - 1:
        raise RuntimeError("mask_rcnn_loss: %d images of proposals but %d packed images"
                           % (len(num_proposals), len(packed.image_start) - 1))
    out = []
    for i, k in enumerate(num_proposals):
        off, g = packed.image_start[i], packed.image_start[i + 1] - packed.image_start[i]
        mi = (torch.arange(k, device=device) if mask_index is None else mask_index[i].to(device=device, dtype=torch.int64))
        out.append(torch.where((mi >= 0) & (mi < g), mi + off, torch.full_like(mi, -1)))
    return torch.cat(out) if out else torch.zeros((0,), dtype=torch.int64, device=device)
