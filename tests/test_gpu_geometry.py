"""The flood kernel across the fields of view, depths, grids and chain counts the engine accepts.

Every other GPU test runs the conv stack at fov (33, 33, 33) / depth 12 or (17, 33, 33) / depth 9 on the default
grid.  Here:

a. ffn_predict in all three compute modes against the float64 oracle at every (FoV, depth) of
   tests/test_geometry_oracle.py:SWEEP, with the bounds of tests/test_gpu_parity.py: fp32 and split fp16
   <= 1e-4; fp16 <= 1.5e-2 against the fp16-operand oracle and <= 4e-2 against float64.  Depth 16 keeps these
   bounds: on the CPU its fp32- and float64-accumulate fp16-operand oracles differ by 5.6e-3 at most (7.6e-3 at
   depth 12 on the golden patches, where the kernel measures 7.8e-3), and the fp16-operand float64 oracle is within
   1.0e-2 of float64 (2.6e-2 at depth 12); test_geometry_oracle.py checks that headroom at every depth of the sweep.
b. Logits that do not depend on the grid (set_grid) or the chain count (set_chains): each tile's MMAs and epilogue
   are the same whichever CTA runs them.
c. The device flood-fill loop against the hybrid oracle (the CPU loop driven by the same device network) at three
   more geometries, with chains and a one-CTA grid.
d. Engine creation rejects what it cannot run, and DeviceCanvas.add_id_offset.
"""

import numpy as np
import pytest
import torch

from oracle import flood_fill as ff
from test_geometry_oracle import SWEEP, TOL_FP16, TOL_FP16_OP, TOL_FP32, sweep_patches, sweep_weights

pytestmark = pytest.mark.gpu

TILE_OUT = 126   # FoV rows per tile (kTileOut)


def _modes():
  from ffn_b200 import _lib
  return {'tc': _lib.COMPUTE_FP16_TC, 'fp32': _lib.COMPUTE_FP32, 'x2': _lib.COMPUTE_FP16X2_TC}


def _deltas(fov):
  return tuple(min(8, f // 2) for f in fov)


def _worst(got, want, fov):
  """Where the largest error sits: patch, (z, y, x), its row in the kernel's row space and its tile."""
  d = np.abs(got.astype(np.float64) - want.astype(np.float64)).reshape((-1,) + tuple(fov))
  p, z, y, x = (int(v) for v in np.unravel_index(int(np.argmax(d)), d.shape))
  row = z * (fov[1] + 1) * fov[2] + y * fov[2] + x
  return float(d.max()), 'max |err| %.3g at patch %d, (z, y, x) = (%d, %d, %d), row %d, tile %d' % (
      d.max(), p, z, y, x, row, row // TILE_OUT)


@pytest.mark.parametrize('case', [c[0] for c in SWEEP])
def test_conv_stack_vs_fp64_oracle(golden_dir, case):
  from ffn_b200 import engine as eng
  from oracle.network import ConvStackOracle
  _, fov, depth, kind = next(c for c in SWEEP if c[0] == case)
  w, b = sweep_weights(golden_dir, depth, kind)
  n = 1 if np.prod(fov) > 33 ** 3 else (3 if max(fov) > 17 else 4)
  seeds, imgs = sweep_patches(fov, n)
  want64 = ConvStackOracle(w, b, dtype=torch.float64)(seeds, imgs)
  want16 = ConvStackOracle(w, b, dtype=torch.float64, operand_round='fp16')(seeds, imgs)
  report = []
  for name, mode in _modes().items():
    e = eng.Engine(w, b, fov, _deltas(fov), compute_mode=mode)
    got = e.predict(seeds, imgs)
    info = e.info()
    e.close()
    assert np.isfinite(got).all(), (case, name)
    err64, where64 = _worst(got, want64, fov)
    report.append('%s: vs fp64 %s' % (name, where64))
    if name == 'tc':
      err16, where16 = _worst(got, want16, fov)
      report.append('tc: vs fp16-operand oracle %s' % where16)
      assert err16 <= TOL_FP16_OP and err64 <= TOL_FP16, (case, info['tiles'], report)
    else:
      assert err64 <= TOL_FP32, (case, info['tiles'], report)
  print('%s (%d tiles, batch %d): %s' % (case, info['tiles'], n, '; '.join(report)))


@pytest.mark.parametrize('fov,depth', [((33, 33, 33), 12), ((17, 33, 17), 4)])
def test_logits_do_not_depend_on_grid_or_chains(golden_dir, fov, depth):
  """(33, 33, 33): 294 tiles; (17, 33, 17): 78 tiles, fewer than the SMs.  fp16: every grid x chain count gives the
  default configuration's logits bit for bit; fp32 and split fp16 (one chain at a time): every grid does."""
  from ffn_b200 import engine as eng
  w, b = sweep_weights(golden_dir, depth, 'fib25')
  seeds, imgs = sweep_patches(fov, 5)
  for name, mode in _modes().items():
    e = eng.Engine(w, b, fov, _deltas(fov), compute_mode=mode)
    info = e.info()
    nt = info['tiles']
    ref = e.predict(seeds, imgs)
    assert np.isfinite(ref).all()
    grids = sorted({1, 7, min(61, nt), min(nt, 131, info['sm_count'])}) + [0]
    for grid in grids:
      e.set_grid(grid)
      for chains in ((1, 2, 3, 4) if name == 'tc' else (0,)):
        e.set_chains(chains)
        got = e.predict(seeds, imgs)
        if not np.array_equal(got, ref):
          _, where = _worst(got, ref, fov)
          pytest.fail('%s fov %r: grid %d, %d chains differ from the default configuration: %s' % (
              name, fov, grid, chains, where))
    e.close()


# name: fov, deltas, phantom shape, phantom seed, min_segment_size (the geometries of the toy_geometry fixture)
FLOOD = {
    'g9': ((9, 17, 25), (2, 4, 6), (40, 64, 72), 21, 1000),
    'g5': ((5, 33, 33), (0, 8, 8), (40, 64, 72), 22, 1000),
    'g3': ((3, 3, 3), (1, 1, 1), (12, 14, 16), 23, 100),             # one-voxel moves: a small canvas
}


def _flood_net(golden_dir):
  """FIB-25's first three modules and conv_lom, with the conv_lom bias raised by 5 so that objects grow at these
  small fields of view (unchanged, the truncated network never moves).  Logits stay below ~60."""
  w, b = sweep_weights(golden_dir, 3, 'fib25')
  return w, b[:-1] + [b[-1] + np.float32(5.0)]


def _image(vol):
  return (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)


@pytest.mark.parametrize('name', sorted(FLOOD))
def test_device_loop_bit_exact_vs_hybrid_oracle_at_other_geometries(golden_dir, name):
  from ffn_b200 import _lib, engine as eng
  from ffn_b200.synthetic import voronoi_phantom
  fov, deltas, shape, pseed, min_size = FLOOD[name]
  w, b = _flood_net(golden_dir)
  vol = voronoi_phantom(shape, seed=pseed, cell_volume=30000.0)
  seeds = ff.grid_seeds(shape, step=8, offsets=(0, 4))
  opts = dict(min_segment_size=min_size, min_boundary_dist_zyx=(1, 2, 1))
  for mode in ('tc', 'fp32'):
    e = eng.Engine(w, b, fov, deltas, compute_mode=_modes()[mode])
    e.set_chains(1)
    cv = eng.DeviceCanvas(e, vol, eng.make_options(**opts), 128.0, 33.0)
    origins, overlaps, ctr = cv.segment_all(seeds)
    hyb = ff.Canvas(lambda s, im: e.predict(s, im), _image(vol), fov, deltas,
                    ff.Options(min_segment_size=min_size, min_boundary_dist=(1, 2, 1)))
    hyb.segment_all(seeds)
    seg = cv.read(_lib.ARRAY_SEGMENTATION)
    np.testing.assert_array_equal(seg, hyb.segmentation)
    np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEED), hyb.seed)
    qd = np.abs(cv.read(_lib.ARRAY_QPROB).astype(int) - hyb.seg_prob.astype(int))
    assert qd.max() <= 1 and (qd > 0).mean() < 1e-3                    # expf vs scipy expit at bin edges
    assert ctr.inference_calls == len(hyb.trace)
    assert [(o.id, tuple(o.start_zyx), o.iters) for o in origins] == \
        [(k, v[0], v[1]) for k, v in sorted(hyb.origins.items())]
    for k, v in hyb.overlaps.items():
      assert sorted((o.other_id, o.count) for o in overlaps if o.id == k) == sorted(zip(v[0].tolist(), v[1].tolist()))
    assert ctr.skip_threshold == hyb.counters['skip_threshold']
    assert ctr.skip_invalid_pos == hyb.counters['skip_invalid_pos']
    assert ctr.invalid_small == hyb.counters['invalid-small']
    assert len(origins) >= 1 and max(o.iters for o in origins) > 1       # objects grow
    print('%s %s: %d steps, %d objects, %d rejected' % (name, mode, ctr.inference_calls, len(origins),
                                                        int((seg == -1).sum())))
    cv.close()

    if mode == 'tc':                   # chains: the same result bit for bit
      one = _segment_all_state(e, vol, seeds, 1, opts)
      np.testing.assert_array_equal(one['seg'], seg)
      for chains in (2, 4):
        many = _segment_all_state(e, vol, seeds, chains, opts)
        for k in ('seg', 'seed', 'qprob'):
          np.testing.assert_array_equal(many[k], one[k], err_msg='%d chains: %s' % (chains, k))
        for k in ('origins', 'overlaps', 'ctr'):
          assert many[k] == one[k], (chains, k)
      # one object on a one-CTA grid
      start = tuple(int(v) for v in origins[0].start_zyx)
      e.set_grid(1)
      e.set_chains(0)
      cv = eng.DeviceCanvas(e, vol, eng.make_options(**opts), 128.0, 33.0)
      st = cv.segment_at(start)
      h1 = ff.Canvas(lambda s, im: e.predict(s, im), _image(vol), fov, deltas, ff.Options())
      assert st.iters == h1.segment_at(start) and st.iters > 1
      np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEED), h1.seed)
      cv.close()
      e.set_grid(0)
    e.close()


def _segment_all_state(e, vol, seeds, chains, opts):
  from ffn_b200 import _lib, engine as eng
  e.set_chains(chains)
  cv = eng.DeviceCanvas(e, vol, eng.make_options(**opts), 128.0, 33.0)
  origins, overlaps, ctr = cv.segment_all(seeds)
  out = dict(seg=cv.read(_lib.ARRAY_SEGMENTATION), seed=cv.read(_lib.ARRAY_SEED), qprob=cv.read(_lib.ARRAY_QPROB),
             origins=[(o.id, tuple(o.start_zyx), o.iters) for o in origins],
             overlaps=sorted((o.id, o.other_id, o.count) for o in overlaps),
             ctr={n: getattr(ctr, n) for n, _ in ctr._fields_ if n not in ('device_seconds', 'kernel_launches')})
  cv.close()
  e.set_chains(0)
  return out


def test_engine_rejects_what_it_cannot_run(golden_dir):
  """fx = 33 is the widest x whose stage fits the 227 KB a CTA may opt into; fx = 35 and depth 17 fail on the host
  with their message, before any launch.  The engine is usable afterwards."""
  from ffn_b200 import engine as eng
  w, b = sweep_weights(golden_dir, 2, 'fib25')
  e = eng.Engine(w, b, (3, 3, 33), (1, 1, 8))
  optin = getattr(torch.cuda.get_device_properties(0), 'shared_memory_per_block_optin', 232448)
  assert e.info()['smem_bytes'] <= optin
  e.close()
  with pytest.raises(RuntimeError, match='field of view too large for the shared-memory operand staging'):
    eng.Engine(w, b, (3, 3, 35), (1, 1, 8))
  w17, b17 = sweep_weights(golden_dir, 17, 'fib25')
  with pytest.raises(RuntimeError, match='unsupported depth'):
    eng.Engine(w17, b17, (9, 9, 9), (2, 2, 2))
  w16, b16 = sweep_weights(golden_dir, 16, 'fib25')
  e = eng.Engine(w16, b16, (3, 3, 3), (1, 1, 1))
  seeds, imgs = sweep_patches((3, 3, 3), 1)
  assert np.isfinite(e.predict(seeds, imgs)).all() and e.info()['launches'] == 1
  e.close()


def test_add_id_offset(golden_dir):
  """relabel_offset_kernel (grid-stride loop) on a canvas whose voxel count is not a multiple of the launch stride:
  exactly the ids > 0 move by the offset; -1 markers and zeros stay."""
  from ffn_b200 import _lib, engine as eng
  w, b = sweep_weights(golden_dir, 1, 'fib25')
  e = eng.Engine(w, b, (3, 3, 3), (1, 1, 1))
  shape = (37, 91, 83)                                                  # 279 461 voxels
  stride = e.info()['sm_count'] * 8 * 256
  assert np.prod(shape) % stride != 0 and np.prod(shape) > stride
  cv = eng.DeviceCanvas(e, np.zeros(shape, np.float32), eng.make_options())
  rng = np.random.RandomState(0)
  seg = rng.randint(-1, 5000, size=shape).astype(np.int32)
  seg[rng.rand(*shape) < 0.3] = 0
  seg.reshape(-1)[-1] = 7                                               # the last voxel is a positive id
  cv.write(_lib.ARRAY_SEGMENTATION, seg)
  cv.add_id_offset(1000)
  want = np.where(seg > 0, seg + 1000, seg)
  np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEGMENTATION), want)
  assert (seg == -1).any() and (seg == 0).any()
  cv.close()
  e.close()
