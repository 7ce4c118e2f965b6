"""Cold-path (load-time) resampling of position embeddings.

``interpolate_pos_embeddings`` mirrors tfimm/layers/transformers.py:13-47, which calls
``tf.image.resize(method="bicubic")``.  With ``antialias=False`` that dispatches to the ``ResizeBicubic`` op
with ``half_pixel_centers=True`` (tensorflow/core/kernels/image/resize_bicubic_op.cc): Keys cubic kernel with
A = -0.5 read from a 1024-step table (the fractional source offset is rounded to the table grid), float32
source coordinate ``(o + 0.5) * scale - 0.5`` and -- unlike OpenCV / PyTorch -- taps that fall outside the image
get weight zero with the remaining weights renormalised.  It runs once per weight load on a (1, N, D) tensor, so
it is plain torch on whatever device the weight lives on.
"""
from typing import Tuple

import numpy as np
import torch

_TABLE = 1024
_A = -0.5


def _resize_matrix(n_in: int, n_out: int, dtype, device) -> torch.Tensor:
    """(n_out, n_in) interpolation matrix of TF2's bicubic resize along one axis."""
    x = np.arange(_TABLE + 1, dtype=np.float64) / _TABLE
    near = (((_A + 2.0) * x - (_A + 3.0)) * x * x + 1.0).astype(np.float32)
    x1 = x + 1.0
    far = (((_A * x1 - 5.0 * _A) * x1 + 8.0 * _A) * x1 - 4.0 * _A).astype(np.float32)
    scale = np.float32(n_in) / np.float32(n_out)
    src = (np.arange(n_out, dtype=np.float32) + np.float32(0.5)) * scale - np.float32(0.5)
    base = np.floor(src).astype(np.int64)
    off = np.rint((src - base.astype(np.float32)) * np.float32(_TABLE)).astype(np.int64)
    w = np.zeros((n_out, n_in), dtype=np.float32)
    rows = np.arange(n_out)
    for k, tap in ((-1, far[off]), (0, near[off]), (1, near[_TABLE - off]), (2, far[_TABLE - off])):
        idx = base + k
        ok = (idx >= 0) & (idx < n_in)
        np.add.at(w, (rows[ok], idx[ok]), tap[ok])
    w = w / w.sum(axis=1, keepdims=True, dtype=np.float32)
    return torch.from_numpy(w).to(device=device, dtype=dtype)


def tf_bicubic_resize(images: torch.Tensor, size: Tuple[int, int]) -> torch.Tensor:
    """``tf.image.resize(images, size, method="bicubic")`` for NHWC tensors."""
    _, h, w, _ = images.shape
    mh = _resize_matrix(h, size[0], images.dtype, images.device)
    mw = _resize_matrix(w, size[1], images.dtype, images.device)
    out = torch.einsum("oh,bhwc->bowc", mh, images)
    return torch.einsum("pw,bowc->bopc", mw, out)


def tf_bilinear_resize(images: torch.Tensor, size: Tuple[int, int]) -> torch.Tensor:
    """``tf.image.resize(images, size, method="bilinear")`` for NHWC tensors (``antialias=False``: the ResizeBilinear op
    with ``half_pixel_centers=True``, source coordinate ``(o + 0.5) * scale - 0.5`` clamped to the image), which is
    PyTorch's ``align_corners=False`` bilinear interpolation."""
    x = torch.nn.functional.interpolate(images.permute(0, 3, 1, 2), size=tuple(size), mode="bilinear",
                                        align_corners=False)
    return x.permute(0, 2, 3, 1).contiguous()


def interpolate_pos_embeddings(pos_embed: torch.Tensor, src_grid_size, tgt_grid_size, nb_tokens: int = 0):
    """(1, nb_tokens + h*w, D) -> (1, nb_tokens + h'*w', D); token embeddings are kept as they are."""
    src_grid_size, tgt_grid_size = tuple(src_grid_size), tuple(tgt_grid_size)
    if src_grid_size == tgt_grid_size:
        return pos_embed
    grid = pos_embed[:, nb_tokens:].reshape(1, *src_grid_size, -1)
    grid = tf_bicubic_resize(grid, tgt_grid_size)
    grid = grid.reshape(1, tgt_grid_size[0] * tgt_grid_size[1], -1)
    return torch.cat((pos_embed[:, :nb_tokens], grid), dim=1)
