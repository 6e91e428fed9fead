"""Engines and canvases created and destroyed over and over give the same results and leave no device memory behind.

Each cycle creates an engine, runs predict at batch 1, 8 and 2 (the staging is allocated, grows once, then is reused),
creates a canvas with probability maps, sets and clears both masks, arms the event trace twice at different
capacities and turns it off again (a traced segment_all runs one chain only), runs segment_all on four chains (which
allocates the extra object buffers), and closes the engine before the canvas.
"""

import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FOV, DELTAS = (33, 33, 33), (8, 8, 8)
CYCLES = 10


def _process_device_memory():
  """Device memory NVML reports for this process, summed over the GPUs; None when NVML does not list the process."""
  from cuda.bindings import nvml
  try:
    nvml.init_v2()
  except Exception:  # pylint: disable=broad-except
    return None
  try:
    used = None
    for i in range(nvml.device_get_count_v2()):
      procs = nvml.device_get_compute_running_processes_v3(nvml.device_get_handle_by_index_v2(i))
      for k in range(len(procs)):
        if int(procs[k].pid) == os.getpid():
          used = (used or 0) + int(procs[k].used_gpu_memory)
    return used
  except Exception:  # pylint: disable=broad-except
    return None
  finally:
    nvml.shutdown()


def _cycle(w, b, vol, seeds, patches):
  from ffn_b200 import _lib, engine as eng
  e = eng.Engine(w, b, FOV, DELTAS, compute_mode=_lib.COMPUTE_FP16_TC)
  e.set_chains(4)
  logits = [e.predict(patches[0][:n], patches[1][:n]) for n in (1, 8, 2)]
  cv = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0, keep_probability_maps=True)
  mask = np.zeros(vol.shape, bool)
  mask[:, 32:40, :] = True
  for which in (_lib.MASK_MOVEMENT, _lib.MASK_SEED):
    cv.set_mask(which, mask)
    cv.set_mask(which, None)
  cv.start_trace(1 << 12)
  cv.start_trace(1 << 14)
  cv.start_trace(0)
  cv.segment_all(seeds)
  chains = cv.spec_stats()['chains']
  e.close()   # the canvas keeps the engine alive until it is closed too
  labels = cv.read(_lib.ARRAY_SEGMENTATION)
  qprob = cv.read(_lib.ARRAY_QPROB)
  cv.close()
  return dict(logits=logits, labels=labels, qprob=qprob, chains=chains)


@pytest.fixture(scope='module')
def cycles(golden_dir):
  from ffn_b200 import tf_checkpoint
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))
  g = np.load(os.path.join(golden_dir, 'flood_fill_64.npz'))
  rng = np.random.RandomState(0)
  patches = (rng.uniform(0.0, 1.0, (8,) + FOV).astype(np.float32), rng.randn(8, *FOV).astype(np.float32))
  results, memory = [], []
  for _ in range(CYCLES):
    results.append(_cycle(w, b, g['volume'], g['seeds'], patches))
    memory.append(_process_device_memory())
  return results, memory


def test_every_cycle_gives_the_same_results(cycles):
  results, _ = cycles
  first = results[0]
  assert first['chains'] == 4
  assert len(np.unique(first['labels'])) > 2
  for r in results[1:]:
    assert r['chains'] == 4
    for got, want in zip(r['logits'], first['logits']):
      np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(r['labels'], first['labels'])
    np.testing.assert_array_equal(r['qprob'], first['qprob'])
  # predict at batch 2 after batch 8 reuses the larger staging: the same patches give the same logits
  np.testing.assert_array_equal(first['logits'][2], first['logits'][1][:2])


def test_device_memory_returns_to_the_first_cycle_level(cycles):
  _, memory = cycles
  print('device memory of this process after each cycle (bytes, NVML):', memory)
  if any(m is None for m in memory):
    pytest.skip('NVML lists no compute process with pid %d (in a container NVML may report the process under another '
                'pid), or NVML is unavailable: memory not checked' % os.getpid())
  assert memory[-1] <= memory[0], memory


def test_a_smaller_engine_leaves_a_larger_ones_launches_alone(golden_dir):
  """An engine of a smaller field of view created after a larger one must not lower what the larger one's flood-kernel
  launches may use: the larger engine's predict and segment_at give what they gave before the smaller one existed."""
  from ffn_b200 import _lib, engine as eng, tf_checkpoint
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))
  vol = np.load(os.path.join(golden_dir, 'flood_fill_64.npz'))['volume']
  rng = np.random.RandomState(1)
  seed, image = rng.uniform(0.0, 1.0, (2,) + FOV).astype(np.float32), rng.randn(2, *FOV).astype(np.float32)
  large = eng.Engine(w, b, FOV, DELTAS, compute_mode=_lib.COMPUTE_FP16_TC)

  def run():
    logits = large.predict(seed, image)
    cv = eng.DeviceCanvas(large, vol, eng.make_options(), 128.0, 33.0)
    steps = cv.segment_at((16, 48, 32), max_steps=6).iters
    out = cv.read(_lib.ARRAY_SEED)
    cv.close()
    return logits, steps, out

  before = run()
  small = eng.Engine(w, b, (3, 3, 3), (1, 1, 1), compute_mode=_lib.COMPUTE_FP16_TC)
  after = run()
  small.close()
  large.close()
  assert after[1] == before[1] == 6
  np.testing.assert_array_equal(after[0], before[0])
  np.testing.assert_array_equal(after[2], before[2])
