"""Consensus of two segmentations of one subvolume (ffn/inference/consensus.py:30-96).

Split consensus keeps a segment of the first segmentation only where the second agrees with it: every overlap of
two segments becomes a segment of its own, the largest overlap keeping the first segmentation's id.  Computing it
between a forward and a reverse seed-order run lowers the false-merge rate.  The intersection runs on the device
(`segmentation.split_segmentation_by_intersection`).
"""

import numpy as np

from . import consensus_pb2
from . import segmentation
from . import storage


def compute_consensus_for_segmentations(v1, v2, request, device: int = 0):
  """Consensus of two segmentations (consensus.py:30-54).

  Args:
    v1: 1st segmentation as a 3d uint64 ndarray; modified in place
    v2: 2nd segmentation as a 3d uint64 ndarray
    request: ConsensusRequest proto
    device: CUDA device index (an H100)

  Returns:
    3d consensus segmentation array, in the smallest unsigned dtype that holds its ids

  Raises:
    ValueError: if an unsupported consensus type is requested
  """
  if request.type == consensus_pb2.ConsensusRequest.CONSENSUS_SPLIT:
    segmentation.split_segmentation_by_intersection(v1, v2, request.split_min_size, device=device)
    v1 = segmentation.reduce_id_bits(v1)
  else:
    raise ValueError('Unsupported mode: %s' % request.type)
  return v1


def compute_consensus(corner, request, device: int = 0):
  """Consensus segmentation of two FFN subvolumes (consensus.py:57-96).

  Args:
    corner: lower corner of the subvolume as a (z, y, x) tuple
    request: ConsensusRequest proto; both sources need `split_cc: false` (see
      `storage.load_segmentation_from_source`)
    device: CUDA device index (an H100)

  Returns:
    tuple of:
      consensus segmentation as a z, y, x uint numpy array
      origin dictionary of the consensus segmentation: the first segmentation's origin of every non-zero id still
      present (a new id that equals one of its origin keys keeps that origin, as in the reference)
  """
  v1, v1_origins = storage.load_segmentation_from_source(request.segmentation1, corner)
  v2, _ = storage.load_segmentation_from_source(request.segmentation2, corner)
  v1 = compute_consensus_for_segmentations(v1, v2, request, device=device)
  relabeled_origins = {}
  for seg_id in np.unique(v1):
    if seg_id == 0:
      continue
    if seg_id in v1_origins:
      relabeled_origins[seg_id] = v1_origins[seg_id]
  return v1, relabeled_origins
