"""Numpy restatement of split consensus (ffn/inference/segmentation.py:181-290, consensus.py:30-96).

Every overlapping (id_a, id_b) pair of voxels is one segment.  In (id_b, id_a) order, a pair maps to 0 when it has
fewer than `min_size` voxels or id_a == 0, to id_a when id_b is id_a's largest overlap (the smallest id_b among equal
counts), and otherwise to the next new id after max(a).  Vectorised with np.unique and a lexsort; it shares no code
with the device path or the reference's per-pair loop.
"""

import numpy as np


def split_segmentation_by_intersection(a, b, min_size):
  """Rewrites uint64 `a` in place; `b` is not changed."""
  if a.shape != b.shape:
    raise ValueError('shape mismatch')
  if a.dtype != np.uint64:
    raise TypeError('a must be uint64')
  if a.size == 0:
    raise ValueError('empty')
  if b.dtype != np.uint64:
    raise TypeError('b must be uint64')
  ids_a, rank_a = np.unique(a, return_inverse=True)
  ids_b, rank_b = np.unique(b, return_inverse=True)
  # ranks keep the order of the ids, so these keys sort b-major, a-minor like the ids themselves
  key = rank_b.reshape(-1).astype(np.uint64) << np.uint64(32) | rank_a.reshape(-1).astype(np.uint64)
  pairs, inverse, counts = np.unique(key, return_inverse=True, return_counts=True)
  pa = ids_a[(pairs & np.uint64(0xFFFFFFFF)).astype(np.int64)]
  pb = ids_b[(pairs >> np.uint64(32)).astype(np.int64)]
  # per id_a: the largest count, then the smallest id_b
  order = np.lexsort((pb, -counts, pa))
  head = np.ones(order.size, bool)
  head[1:] = pa[order][1:] != pa[order][:-1]
  partner = np.zeros(pairs.size, bool)
  partner[order[head]] = True
  dropped = (counts < min_size) | (pa == 0)
  new = ~dropped & ~partner
  max_id = int(a.max())
  n_new = int(new.sum())
  if max_id + n_new > 2**64 - 1:
    raise OverflowError('new ids do not fit in 64 bits')
  new_ids = np.uint64(max_id) + np.cumsum(new, dtype=np.uint64)
  labels = np.where(dropped, np.uint64(0), np.where(partner, pa, new_ids))
  a.reshape(-1)[...] = labels[inverse.reshape(-1)]


def reduce_id_bits(seg):
  m = int(seg.max())
  for dt in (np.uint8, np.uint16, np.uint32):
    if m <= np.iinfo(dt).max:
      return seg.astype(dt)
  return seg


def compute_consensus_for_segmentations(v1, v2, split_min_size, consensus_type=2):
  """CONSENSUS_SPLIT (2) only; `v1` is modified in place and the result has the smallest unsigned dtype."""
  if consensus_type != 2:
    raise ValueError('Unsupported mode: %s' % consensus_type)
  split_segmentation_by_intersection(v1, v2, split_min_size)
  return reduce_id_bits(v1)


def relabeled_origins(v1, origins):
  """The origins of the non-zero ids present in the consensus segmentation `v1`."""
  present = set(int(x) for x in np.unique(v1)) - {0}
  return {k: v for k, v in origins.items() if int(k) in present}
