"""Partition map on the device (ffn_compute_partitions): against the reference's own function
(tests/golden/partitions_ref.npz), against the numpy oracle on Voronoi phantoms across radii, label dtypes and
scratch budgets, and end to end through the compute_partitions.py script."""

import numpy as np
import pytest
from google.protobuf import text_format

import compute_partitions as script
from ffn_b200 import partitions
from ffn_b200 import synthetic
from ffn_b200.inference import inference_pb2
from ffn_b200.inference import storage
from oracle import partitions as op

pytestmark = pytest.mark.gpu

from test_partitions import assert_matches, call, case_ids, fixture, reference_cases  # noqa: E402

THRESHOLDS = [0.025, 0.05, 0.075, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]
SHAPE = (128, 160, 144)
MASK = 'masks { coordinate_expression { expression: "(x - 2 * y > 100) | (z == 70)" } }'
REGIONS = [(20, 30, 40, 12), (150.5, 10, 64, 20.25), (70, 80, 140, 30)]


@pytest.mark.parametrize('idx', range(len(case_ids())), ids=case_ids())
@pytest.mark.parametrize('scratch_bytes', [0, 1])
def test_device_equals_reference(idx, scratch_bytes, tmp_path):
  c = reference_cases(tmp_path)[idx]

  def device(*args):
    pm = partitions.partition_map(*args, scratch_bytes=scratch_bytes)
    return pm.corner, pm.partitions
  seg, res = call(device, c)
  assert_matches(c, seg, res)


@pytest.fixture(scope='module')
def phantom():
  _, cells = synthetic.voronoi_phantom(SHAPE, 11, return_cells=True)
  return cells


def relabel(cells, dtype):
  """The phantom's ids (0 kept) mapped injectively into `dtype`, towards its extremes."""
  ids = np.unique(cells)
  assert ids[0] == 0 and ids.size < 200
  k = np.arange(1, ids.size, dtype=np.int64)
  table = {
      np.uint8: k + 50,
      np.uint16: 65535 - k * 7,
      np.int32: np.where(k % 2 == 1, -k * 1000, k * 1000 + 2**30),
      np.int64: np.where(k % 3 == 0, -2**63 + k, k * 2**40),
      np.uint64: (np.uint64(2**64 - 1) - k.astype(np.uint64) * np.uint64(2**61 // 200)),
  }[dtype]
  lut = np.zeros(int(ids.max()) + 1, dtype)
  lut[ids[1:]] = np.asarray(table).astype(dtype)
  return lut[cells]


_ORACLE = {}


def oracle(cells, radius):
  if radius not in _ORACLE:
    configs = inference_pb2.MaskConfigs()
    text_format.Parse(MASK, configs)
    mask = storage.build_mask(configs.masks, (0, 0, 0), cells.shape)
    seg = cells.astype(np.int64)
    _ORACLE[radius] = op.compute_partitions(seg, THRESHOLDS, list(radius), None, REGIONS, mask, 1000), seg
  return _ORACLE[radius]


@pytest.mark.parametrize('radius', [(0, 0, 0), (1, 2, 3), (8, 8, 4), (16, 16, 16)], ids=str)
@pytest.mark.parametrize('dtype', [np.uint8, np.uint16, np.int32, np.int64, np.uint64], ids=lambda d: d.__name__)
@pytest.mark.parametrize('scratch_bytes', [0, 1 << 20], ids=['one_group', 'many_groups'])
def test_device_equals_oracle_on_phantoms(phantom, radius, dtype, scratch_bytes):
  (corner, want), dusted = oracle(phantom, radius)
  seg = relabel(phantom, dtype)
  configs = inference_pb2.MaskConfigs()
  text_format.Parse(MASK, configs)
  pm = partitions.partition_map(seg, THRESHOLDS, list(radius), None, REGIONS, configs, 1000,
                                scratch_bytes=scratch_bytes)
  assert (pm.corner == corner).all()
  assert pm.partitions.shape == want.shape and (pm.partitions == want).all(), int((pm.partitions != want).sum())
  assert ((seg == 0) == (dusted == 0)).all()


def test_partition_counts_equal_unique(phantom):
  pm = partitions.partition_map(phantom.copy(), THRESHOLDS, [4, 4, 4], None, REGIONS, None, 1000)
  got = partitions.partition_counts(pm.counts)
  want = np.array(np.unique(pm.partitions, return_counts=True))
  assert got.shape == want.shape and (got == want).all()
  assert pm.counts.sum() == pm.partitions.size


def test_two_calls_equal(phantom):
  a = partitions.partition_map(phantom.copy(), THRESHOLDS, [16, 16, 16], None, None, None, 1000)
  b = partitions.partition_map(phantom.copy(), THRESHOLDS, [16, 16, 16], None, None, None, 1000)
  assert (a.partitions == b.partitions).all() and (a.counts == b.counts).all()


def test_script_equals_reference_main(tmp_path):
  g = fixture()
  src = tmp_path / 'in.npz'
  np.savez(src, **{'stack': g['main_seg'], 'stack.bounding_boxes': g['main_bboxes']})
  dst = tmp_path / 'out.npz'
  argv = [a.replace('in.h5:', '%s:' % src).replace('out.h5:', '%s:' % dst) for a in g['main_argv'].tolist()]
  script.FLAGS(['compute_partitions.py'] + argv)
  script.main([])
  with np.load(dst) as f:
    assert f['af'].dtype == np.uint8 and (f['af'] == g['main_out']).all()
    assert (f['af.bounding_boxes'] == g['main_out_bboxes']).all()
    assert (f['af.partition_counts'] == g['main_partition_counts']).all()
