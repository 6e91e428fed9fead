"""Split consensus on the device (ffn_split_intersection): against the reference's own modules
(tests/golden/consensus_ref.npz), end to end through compute_consensus, and against the numpy oracle on Voronoi
phantoms at the size of the configs[4] volume with ids above 2^32."""

import numpy as np
import pytest

from ffn_b200 import synthetic
from ffn_b200.inference import consensus
from ffn_b200.inference import consensus_pb2
from ffn_b200.inference import segmentation
from oracle import consensus as oc

pytestmark = pytest.mark.gpu

from test_consensus import ERRORS, consensus_cases, plain_origins, split_cases  # noqa: E402


@pytest.mark.parametrize('case', split_cases(), ids=lambda c: c[0])
def test_device_equals_reference(case):
  tag, a, b, min_size, ctype, want, after, error = case
  req = consensus_pb2.ConsensusRequest(split_min_size=min_size)
  if ctype != 2:
    class Req:
      type = ctype
      split_min_size = min_size
    req = Req()
  v1, b_in = a.copy(), b.copy()
  if error:
    with pytest.raises(ERRORS[error]):
      consensus.compute_consensus_for_segmentations(v1, b_in, req)
    return
  got = consensus.compute_consensus_for_segmentations(v1, b_in, req)
  assert got.dtype == want.dtype and (got == want).all(), tag
  assert v1.dtype == np.uint64 and (v1 == after).all(), tag   # a is rewritten in place
  assert (b_in == b).all(), tag                                # b is not


def test_compute_consensus_equals_reference(tmp_path):
  for c in consensus_cases(tmp_path):
    seg, origins = consensus.compute_consensus(c['corner'], c['request'])
    assert seg.dtype == c['seg'].dtype and (seg == c['seg']).all(), c['tag']
    assert plain_origins(origins) == c['origins'], c['tag']
    assert set(c['stale']) <= set(int(k) for k in origins)


def test_non_contiguous_input_is_written_back():
  case = {c[0]: c for c in split_cases()}['min_drop']
  _, a, b, min_size, _, _, after, _ = case
  buf = np.zeros((2,) + a.shape[:2] + (2 * a.shape[2],), np.uint64)
  view, b_view = buf[0, :, :, ::2], buf[1, :, :, ::2]
  view[...] = a
  b_view[...] = b
  segmentation.split_segmentation_by_intersection(view, b_view, min_size)
  assert (view == after).all() and (b_view == b).all() and not buf[:, :, :, 1::2].any()


def test_new_id_overflow_is_checked():
  a = np.array([[[2**64 - 1, 2**64 - 1, 5]]], np.uint64)
  b = np.array([[[1, 2, 1]]], np.uint64)
  with pytest.raises(RuntimeError, match='64 bits'):
    segmentation.split_segmentation_by_intersection(a, b, 0)
  b[...] = 1   # no new id: max(a) stays
  segmentation.split_segmentation_by_intersection(a, b, 0)
  assert a.tolist() == [[[2**64 - 1, 2**64 - 1, 5]]]


@pytest.mark.parametrize('big_in', ['a', 'b'])
def test_device_equals_oracle_at_size(big_in):
  """The configs[4] volume (256x512x512): cells cut along different planes in each input, pairwise merges in the
  second, ids above 2^32 in one input; min_size drops the smallest fragments."""
  a, b = synthetic.consensus_pair((256, 512, 512), seed=3, big_ids=True)
  if big_in == 'b':
    a, b = b, a
  assert max(int(a.max()), int(b.max())) > 2**32
  want = a.copy()
  oc.split_segmentation_by_intersection(want, b, 50)
  b_in = b.copy()
  segmentation.split_segmentation_by_intersection(a, b, 50)
  assert (b == b_in).all()
  assert (a == want).all()
  assert np.unique(want).size > 10000
