"""Deterministic synthetic EM-like volumes (Voronoi-membrane phantom).

The reference's sample volume (training_sample2/grayscale_maps.h5) is not shipped, so every
benchmark/parity configuration uses this generator (contract in SURVEY.md section 8d):

  rng = RandomState(seed); ncell = round(volume / 75000); sites = rng.rand(ncell, 3) * shape
  membrane  <=>  (d2 - d1) < 2.0   (distances to the nearest / 2nd nearest site)
  intensity = where(membrane, 70, 160) + rng.randn(*shape) * 12  -> gaussian blur -> clip -> uint8
"""

from __future__ import annotations

import numpy as np
from scipy import ndimage
from scipy.spatial import cKDTree


def voronoi_phantom(shape_zyx, seed: int, sigma=(1.0, 1.0, 1.0), voxel_size_zyx=(1.0, 1.0, 1.0),
                    return_cells: bool = False, cell_volume: float = 75000.0):
  """Returns a uint8 (z,y,x) volume (and optionally the int32 ground-truth cell ids)."""
  shape = tuple(int(s) for s in shape_zyx)
  rng = np.random.RandomState(seed)
  ncell = max(2, int(round(np.prod(shape) / cell_volume)))
  sites = rng.rand(ncell, 3) * np.asarray(shape, dtype=np.float64)
  scale = np.asarray(voxel_size_zyx, dtype=np.float64)
  tree = cKDTree(sites * scale)

  membrane = np.empty(shape, dtype=bool)
  cells = np.empty(shape, dtype=np.int32) if return_cells else None
  yy, xx = np.meshgrid(np.arange(shape[1]), np.arange(shape[2]), indexing='ij')
  plane = np.stack([np.zeros_like(yy), yy, xx], axis=-1).reshape(-1, 3).astype(np.float64)
  for z in range(shape[0]):
    plane[:, 0] = z
    d, idx = tree.query(plane * scale, k=2, workers=-1)
    membrane[z] = ((d[:, 1] - d[:, 0]) < 2.0).reshape(shape[1], shape[2])
    if return_cells:
      cells[z] = idx[:, 0].reshape(shape[1], shape[2]) + 1

  vol = np.where(membrane, np.float32(70.0), np.float32(160.0))
  # Noise is drawn plane by plane from the same stream so memory stays bounded for 512^3+.
  for z in range(shape[0]):
    vol[z] += (rng.randn(shape[1], shape[2]) * 12.0).astype(np.float32)
  vol = ndimage.gaussian_filter(vol, sigma=sigma, mode='reflect')
  out = np.clip(np.rint(vol), 0, 255).astype(np.uint8)
  if return_cells:
    cells[membrane] = 0
    return out, cells
  return out


def interior_seed(volume_u8: np.ndarray, near_zyx, max_radius: int = 24, bright: int = 140):
  """Snaps `near_zyx` to the closest bright (non-membrane) voxel, deterministic tie-break."""
  z0, y0, x0 = (int(v) for v in near_zyx)
  best = None
  for r in range(max_radius + 1):
    lo = [max(z0 - r, 0), max(y0 - r, 0), max(x0 - r, 0)]
    hi = [min(z0 + r + 1, volume_u8.shape[0]), min(y0 + r + 1, volume_u8.shape[1]),
          min(x0 + r + 1, volume_u8.shape[2])]
    sub = volume_u8[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
    # require a bright 3x3x3 neighbourhood so the seed is not on a membrane
    ok = ndimage.minimum_filter(sub, size=3, mode='nearest') >= bright
    if ok.any():
      zz, yy, xx = np.nonzero(ok)
      d2 = (zz + lo[0] - z0) ** 2 + (yy + lo[1] - y0) ** 2 + (xx + lo[2] - x0) ** 2
      k = int(np.lexsort((xx, yy, zz, d2))[0])
      best = (int(zz[k] + lo[0]), int(yy[k] + lo[1]), int(xx[k] + lo[2]))
      break
  return best if best is not None else (z0, y0, x0)


def consensus_pair(shape_zyx, seed: int = 3, big_ids: bool = False):
  """Two uint64 segmentations of the same Voronoi cells that disagree as a forward and a reverse run do.

  The cells of a 64x128x128 phantom are tiled over `shape_zyx` with distinct ids per tile (membranes stay 0).  The
  first segmentation cuts every cell along one family of parallel planes, the second along another, and the second
  also merges cells pairwise.  With `big_ids`, the first segmentation's ids are scaled above 2^32.
  """
  shape = tuple(int(s) for s in shape_zyx)
  _, cells = voronoi_phantom((64, 128, 128), seed=seed, cell_volume=20000.0, return_cells=True)
  ncell = int(cells.max())
  a = np.zeros(shape, dtype=np.uint64)
  b = np.zeros(shape, dtype=np.uint64)
  z, y, x = np.indices(cells.shape, dtype=np.int64)
  side_a = ((x + 2 * y + 3 * z) // 37) % 2
  side_b = ((2 * x - y + z + 1000) // 29) % 2
  t = 0
  for z0 in range(0, shape[0], 64):
    for y0 in range(0, shape[1], 128):
      for x0 in range(0, shape[2], 128):
        sel = (slice(z0, z0 + 64), slice(y0, y0 + 128), slice(x0, x0 + 128))
        n = tuple(s.stop - s.start if s.stop <= d else d - s.start for s, d in zip(sel, shape))
        c = cells[:n[0], :n[1], :n[2]].astype(np.int64)
        cid = c + t * ncell
        la = np.where(c > 0, 2 * cid + side_a[:n[0], :n[1], :n[2]], 0).astype(np.uint64)
        if big_ids:
          la = np.where(la > 0, la * np.uint64(2**33) + np.uint64(12345), np.uint64(0))
        a[sel] = la
        b[sel] = np.where(c > 0, 2 * (cid // 2) + side_b[:n[0], :n[1], :n[2]] + 1, 0).astype(np.uint64)
        t += 1
  return a, b
