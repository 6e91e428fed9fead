"""Training coordinates on the device (ffn_partition_rows, ffn_coordinate_records): against the reference's own script
(tests/golden/coordinates_ref.npz), the bucketing against np.flatnonzero, the whole pipeline against the numpy oracle
on phantom partition maps, chunking, and end to end through compute_partitions.py and build_coordinates.py."""

import gzip
import io

import numpy as np
import pytest

import build_coordinates as script
import compute_partitions as partition_script
from ffn_b200 import coordinates
from ffn_b200 import partitions
from ffn_b200 import synthetic
from oracle import coordinates as oc

pytestmark = pytest.mark.gpu

from test_coordinates import ERRORS, case_ids, read_coordinates, reference_cases, tfrecord_payloads  # noqa: E402

THRESHOLDS = [0.025, 0.05, 0.075, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]


@pytest.mark.parametrize('idx', range(len(case_ids())), ids=case_ids())
def test_device_equals_reference(idx, tmp_path):
  c = reference_cases()[idx]
  names = [n.encode('utf-8') for n, _ in c['volumes']]
  np.random.seed(c['seed'])
  for k in range(max(c['calls'], 1)):
    out = str(tmp_path / ('coords_%d.gz' % k))
    if c['error']:
      with pytest.raises(ERRORS[c['error']]):
        coordinates.build_coordinates(c['volumes'], c['margin'], out)
      return
    coordinates.build_coordinates(c['volumes'], c['margin'], out)
    centers, got_names = read_coordinates(out)
    assert centers.shape == c['centers'][k].shape and (centers == c['centers'][k]).all()
    assert got_names == [names[i] for i in c['name_index'][k]]


@pytest.fixture(scope='module')
def phantom_maps():
  """Partition maps of two Voronoi phantoms of different shapes (lom_radius 4, the README's thresholds)."""
  maps = []
  for shape, seed in (((48, 64, 56), 3), ((40, 36, 52), 4)):
    _, cells = synthetic.voronoi_phantom(shape, seed, return_cells=True, cell_volume=6000.0)
    pm = partitions.partition_map(cells, THRESHOLDS, [4, 4, 4], min_size=100)
    full = np.full(shape, 255, np.uint8)
    full[4:-4, 4:-4, 4:-4] = pm.partitions
    maps.append(full)
  return maps


def bucketing_inputs(maps):
  rng = np.random.RandomState(7)
  thin = rng.randint(0, 256, (9, 31, 40)).astype(np.uint8)
  return {
      'phantom': (maps[0], (5, 6, 7)),
      'uniform_all_values': (rng.randint(0, 256, (70, 65, 66)).astype(np.uint8), (2, 1, 3)),
      'one_value': (np.full((20, 21, 22), 17, np.uint8), (1, 1, 1)),
      'all_255': (np.full((20, 21, 22), 255, np.uint8), (1, 2, 3)),
      'thin_z': (thin, (4, 2, 2)),
      'thin_y': (thin, (1, 15, 2)),
      'thin_x': (rng.randint(0, 3, (30, 33, 9)).astype(np.uint8), (2, 3, 4)),
      'odd_count': (rng.randint(250, 256, (17, 19, 23)).astype(np.uint8), (1, 1, 1)),   # 15 * 17 * 21 voxels
  }


@pytest.mark.parametrize('name', ['phantom', 'uniform_all_values', 'one_value', 'all_255', 'thin_z', 'thin_y',
                                  'thin_x', 'odd_count'])
def test_bucketing_equals_flatnonzero(phantom_maps, name):
  vol, margin = bucketing_inputs(phantom_maps)[name]
  crop = vol[margin[0]:-margin[0], margin[1]:-margin[1], margin[2]:-margin[2]]
  rows, counts = coordinates.partition_rows(vol, margin, volume_index=3)
  assert (counts == np.bincount(crop.ravel(), minlength=256)).all()
  assert rows.shape == (crop.size - counts[255], 2) and (rows[:, 0] == 3).all()
  start = 0
  for v in range(255):
    want = np.flatnonzero(crop == v)
    assert (rows[start:start + want.size, 1] == want).all(), v
    start += want.size


@pytest.mark.parametrize('seed', [0, 12345])
def test_pipeline_equals_oracle(phantom_maps, seed, tmp_path):
  margin = (6, 5, 7)
  out = str(tmp_path / 'c.gz')
  np.random.seed(seed)
  want, vol = oc.build_coordinates(phantom_maps, margin)
  want_state = np.random.get_state()
  np.random.seed(seed)
  coordinates.build_coordinates([('a', phantom_maps[0]), ('b', phantom_maps[1])], margin, out)
  state = np.random.get_state()
  centers, names = read_coordinates(out)
  assert centers.shape == want.shape and (centers == want).all()
  assert names == [(b'a', b'b')[i] for i in vol]
  assert (state[1] == want_state[1]).all() and state[2:] == want_state[2:]


def _raw(volumes, margin, seed, chunk_rows, path):
  np.random.seed(seed)
  coordinates.build_coordinates(volumes, margin, path, chunk_rows=chunk_rows)
  with open(path, 'rb') as f:
    return gzip.decompress(f.read())


def test_chunk_sizes_give_identical_bytes(tmp_path):
  c = reference_cases()[case_ids().index('non_ascii')]
  small = [_raw(c['volumes'], c['margin'], 5, n, str(tmp_path / 'c.gz')) for n in (1, 7, 4099, coordinates.CHUNK_ROWS)]
  assert all(s == small[0] for s in small) and len(small[0]) > 0
  c = reference_cases()[case_ids().index('large')]
  big = [_raw(c['volumes'], c['margin'], 5, n, str(tmp_path / 'c.gz')) for n in (7, 4099, coordinates.CHUNK_ROWS)]
  assert all(s == big[0] for s in big)


def test_two_calls_equal(phantom_maps, tmp_path):
  vols = [('a', phantom_maps[0]), ('b', phantom_maps[1])]
  assert _raw(vols, (4, 4, 4), 9, coordinates.CHUNK_ROWS, str(tmp_path / 'a.gz')) == \
      _raw(vols, (4, 4, 4), 9, coordinates.CHUNK_ROWS, str(tmp_path / 'b.gz'))


def test_only_255_raises_as_reference(tmp_path):
  out = str(tmp_path / 'c.gz')
  with pytest.raises(ValueError):
    coordinates.build_coordinates([('a', np.full((8, 8, 8), 255, np.uint8))], (1, 1, 1), out)


def test_record_known_answer():
  # center [300, 5, 70000], name b'vol': one record of a crop whose last voxel is that center (margin 0).
  table_rows = np.array([[0, (70000 * 6 + 5) * 301 + 300]], np.int64)
  fd = io.BytesIO()
  coordinates.write_records(fd, table_rows, ['vol'], [(70001, 6, 301)], (0, 0, 0))
  raw = gzip.decompress(fd.getvalue())
  payload = bytes.fromhex('0a340a140a0663656e746572120a1a080a06ac0205f0a2040a1c0a116c6162656c5f766f6c756d655f6e616d65'
                          '12070a050a03766f6c')
  assert tfrecord_payloads(raw) == [payload]
  assert len(raw) == 16 + 54


def test_script_end_to_end(tmp_path):
  _, cells = synthetic.voronoi_phantom((40, 44, 48), 2, return_cells=True, cell_volume=5000.0)
  np.savez(tmp_path / 'gt.npz', stack=cells)
  partition_script.FLAGS(['compute_partitions.py', '--input_volume=%s:stack' % (tmp_path / 'gt.npz'),
                          '--output_volume=%s:af' % (tmp_path / 'af.npz'), '--thresholds=0.1,0.3,0.5,0.7,0.9',
                          '--lom_radius=3,3,3', '--min_size=50'])
  partition_script.main([])
  with np.load(tmp_path / 'af.npz') as f:
    af = f['af']
  out = str(tmp_path / 'coords.gz')
  af_path = tmp_path / 'af.npz'
  script.FLAGS(['build_coordinates.py', '--partition_volumes=train:%s:af,again:%s:af' % (af_path, af_path),
                '--coordinate_output=%s' % out, '--margin=4,5,6'])
  np.random.seed(21)
  script.main([])
  np.random.seed(21)
  want, vol = oc.build_coordinates([af, af], (4, 5, 6))
  centers, names = read_coordinates(out)
  assert centers.shape == want.shape and (centers == want).all()
  assert names == [(b'train', b'again')[i] for i in vol]
