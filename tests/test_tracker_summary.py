"""TensorBoard event files (ffn_b200/training/summary.py): CRC-32C, the round trip through the project's reader and
TensorBoard's, and train.py's summary timing and tracker reset with a stand-in trainer.  CPU only."""

import json
import os
import subprocess
import sys

import numpy as np
import pytest

from ffn_b200.training import summary
from ffn_b200.training import tracker as tk

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_crc32c_check_value():
  assert summary.crc32c(b'123456789') == 0xE3069283   # RFC 3720, B.4
  assert summary.crc32c(b'') == 0
  assert summary.crc32c(bytes(32)) == 0x8A9136AA      # RFC 3720, B.4: 32 bytes of zeros


def _state():
  rng = np.random.RandomState(0)
  planes = [tuple((np.where(rng.rand(h, w) < 0.5, 0.95, 0.05).astype(np.float32),
                   rng.standard_normal((h, w)).astype(np.float32) * 4) for h, w in ((5, 7), (3, 7), (3, 5)))
            for _ in range(2)]
  return tk.TrackerState(steps=3, fov_voxels=3 * 2 * 27, patches=2, eval_voxels=2 * 105,
                         prediction_counts=np.array([10, 150, 20, 30]), patch_loss=1.25,
                         moves={0: np.array([3, 1, 2]), 2: np.array([0, 4, 0])}, planes=planes,
                         coords=[(0, (10, 11, 12)), (1, (3, 4, 5))])


def test_summaries_formulas():
  got = dict(tk.summaries(_state(), ['a', 'b']))
  assert got['eval/patch_loss'] == 0.625 and got['eval/patches'] == 2
  assert got['eval/all/accuracy'] == 160 / 210 and got['eval/all/precision'] == 10 / 30
  assert got['eval/all/recall'] == 10 / 40 and got['eval/all/specificity'] == 150 / 170
  p, r = 10 / 30, 10 / 40
  assert got['eval/all/f1'] == 2.0 * p * r / (p + r)
  assert got['moves/total'] == 10 and got['moves/all/correct'] == 0.3 and got['moves/all/spurious'] == 0.2
  assert got['moves/r=2/missed'] == 1.0 and got['moves/r=2/total'] == 4 and got['moves/r=0/total'] == 6
  assert got['fov/masked_voxel_fraction'] == 0 and got['fov/average_weight'] == 1 and got['masked_voxel_fraction'] == 0
  img = got['final_xz/1']
  assert (img.height, img.width) == (3, 21)
  assert sorted(t for t in got if t.startswith('final_')) == sorted(
      'final_%s/%d' % (a, i) for a in ('xy', 'xz', 'yz') for i in range(2))


def _write(tmp_path):
  w = summary.EventWriter(str(tmp_path))
  values = tk.summaries(_state(), ['a', 'b'])
  w.add(50, values, wall_time=1.5)
  w.add(100, [('pixel_loss', 0.25)], wall_time=2.5)
  w.close()
  return w.path, values


def test_event_file_reads_back(tmp_path):
  path, values = _write(tmp_path)
  assert os.path.basename(path).startswith('events.out.tfevents.')
  events = summary.read_events(path)
  assert events[0].file_version == 'brain.Event:2' and len(events) == 3
  assert [(e.step, e.wall_time) for e in events[1:]] == [(50, 1.5), (100, 2.5)]
  got = {v.tag: v for v in events[1].summary.value}
  for tag, v in values:
    if isinstance(v, tk.Image):
      assert (got[tag].image.height, got[tag].image.width, got[tag].image.colorspace) == (v.height, v.width, 3)
      assert got[tag].image.encoded_image_string == v.png
    else:
      assert got[tag].simple_value == np.float32(v)
  assert events[2].summary.value[0].tag == 'pixel_loss'
  data = bytearray(open(path, 'rb').read())
  data[-6] ^= 1
  open(path, 'wb').write(bytes(data))
  with pytest.raises(ValueError, match='checksum'):
    summary.read_events(path)


def test_event_file_reads_in_tensorboard(tmp_path):
  ea = pytest.importorskip('tensorboard.backend.event_processing.event_accumulator')
  _, values = _write(tmp_path)
  acc = ea.EventAccumulator(str(tmp_path), size_guidance={ea.IMAGES: 0, ea.SCALARS: 0})
  acc.Reload()
  tags = acc.Tags()
  scalars = {t: v for t, v in values if not isinstance(v, tk.Image)}
  assert set(scalars) | {'pixel_loss'} == set(tags['scalars'])
  for t, v in scalars.items():
    (ev,) = acc.Scalars(t)
    assert ev.step == 50 and ev.value == np.float32(v)
  assert acc.Scalars('pixel_loss')[0].step == 100
  images = {t: v for t, v in values if isinstance(v, tk.Image)}
  assert set(images) == set(tags['images'])
  (im,) = acc.Images('final_yz/0')
  assert im.step == 50 and im.encoded_image_string == images['final_yz/0'].png


_TIMING = r'''
import json, sys, tempfile
import numpy as np
import train
from ffn_b200.training import summary, tracker as tk

class Trainer:
  global_step = 0
  def train(self, loop, n):
    self.global_step += n
    return np.arange(self.global_step - n, self.global_step, dtype=np.float64)
  def current_learning_rate(self):
    return np.float32(0.5)
  def weights(self):
    return [np.zeros(1, np.float32)], [np.zeros(1, np.float32)]

class Loop:
  reads = []
  def tracker(self, reset=False):
    self.reads.append(reset)
    p = len(self.reads)
    return tk.TrackerState(steps=50, fov_voxels=50 * 27, patches=p, eval_voxels=p * 27,
                           prediction_counts=np.array([1, 2, 3, 4]), patch_loss=0.5 * p, moves={0: np.array([1, 0, 1])},
                           planes=[], coords=[])

times = iter([0.0, 5.0, 11.0, 12.0, 25.0, 26.0, 27.0, 40.0])   # the start, then one per call boundary
d = tempfile.mkdtemp()
losses = train.run(Trainer(), Loop(), ['v'], d, 7 * train.STEPS_PER_CALL - 10, 10, 1e9, clock=lambda: next(times))
import glob
events = summary.read_events(glob.glob(d + '/events.out.tfevents.*')[0])
print(json.dumps({'n': len(losses), 'reads': Loop.reads,
                  'events': [[e.step, {v.tag: v.simple_value for v in e.summary.value}] for e in events[1:]]}))
'''


def test_train_py_summary_timing(tmp_path):
  """Summaries at the first call boundary after --summary_rate_secs, each reading and resetting the tracker once."""
  res = subprocess.run([sys.executable, '-c', _TIMING], capture_output=True, text=True, cwd=str(tmp_path),
                       env=dict(os.environ, PYTHONPATH=REPO))
  assert res.returncode == 0, res.stderr[-3000:]
  got = json.loads(res.stdout.strip().splitlines()[-1])
  assert got['n'] == 340
  # boundaries at t = 5, 11, 12, 25, 26, 27, 40 after steps 50 .. 340: due at 11 (> 0 + 10), 25 (> 21), 40 (> 35)
  assert got['reads'] == [True, True, True]
  assert [e[0] for e in got['events']] == [100, 200, 340]
  first = got['events'][0][1]
  assert first['eval/patches'] == 1 and first['eval/patch_loss'] == 0.5 and first['pixel_loss'] == 99
  assert first['optimizer_loss'] == 99 and first['learning_rate'] == 0.5
  assert got['events'][2][1]['pixel_loss'] == 339
