"""The CPU oracles at fields of view, deltas and depths other than the flagship (33, 33, 33) / depth 12.

* The flood-fill oracle loop (oracle/flood_fill.py) against the reference's own Canvas.segment_all at three more
  geometries (fixture from tests/golden/make_golden_geometry.py, toy network).
* The power of the conv-stack tolerances of tests/test_gpu_geometry.py: at every (FoV, depth) of its sweep, a
  float64 restatement of the conv stack in the device's row space, with one deliberate arithmetic bug at a
  time, must differ from the correct stack by at least 10x the bound the GPU test applies.  So a kernel that
  drops an x-border mask, reads a dy tap across a z-plane, mixes up the residual stream or adds a bias twice
  cannot pass that test at that geometry.

The sweep table (SWEEP) and its inputs are defined here and shared with the GPU test.
"""

import json
import os

import numpy as np
import pytest
import torch

from oracle import flood_fill as ff
from oracle.toy_net import toy_image, toy_net

# (id, fov_zyx, depth, weights): the geometries and depths tests/test_gpu_geometry.py runs in all compute modes.
# 'fib25' takes the first `depth` modules of FIB-25 (modules repeat beyond 12); 'random' is independent weights.
SWEEP = [
    ('fov3_d1', (3, 3, 3), 1, 'fib25'),
    ('fov9x17x3_d2', (9, 17, 3), 2, 'fib25'),            # fx = 3: two thirds of all rows are x-border rows
    ('fov9x17x25_d3', (9, 17, 25), 3, 'fib25'),
    ('fov3x33x33_d2', (3, 33, 33), 2, 'fib25'),
    ('fov25x33x33_d4', (25, 33, 33), 4, 'fib25'),
    ('fov33x33x31_d5', (33, 33, 31), 5, 'fib25'),
    ('fov65x33x33_d12', (65, 33, 33), 12, 'fib25'),      # 579 tiles: 5 per CTA at 132 CTAs
    ('fov9x17x25_d16', (9, 17, 25), 16, 'fib25'),        # nconv = 32, the most the kernel holds
    ('fov11x13x15_d6_random', (11, 13, 15), 6, 'random'),
]

# Bounds of the GPU test (the bounds of tests/test_gpu_parity.py, kept at every geometry).
TOL_FP32 = 1e-4        # fp32 and split-fp16 modes vs the float64 oracle
TOL_FP16_OP = 1.5e-2   # fp16 mode vs the fp16-operand oracle
TOL_FP16 = 4e-2        # fp16 mode vs the float64 oracle

PAD = float(ff.f32_logit(0.05))
INIT = float(ff.f32_logit(0.95))


def _load(golden_dir, name):
  return np.load(os.path.join(golden_dir, name), allow_pickle=False)


def fib25(golden_dir):
  from ffn_b200 import tf_checkpoint
  return tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))


def sweep_weights(golden_dir, depth, kind):
  """Weight / bias lists (conv0_a, conv0_b, ..., conv_lom) of a `depth`-module network."""
  if kind == 'fib25':
    w, b = fib25(golden_dir)
    mods = [0] + [m if m <= 11 else (m - 1) % 11 + 1 for m in range(1, depth)]
    return ([w[2 * m + i] for m in mods for i in (0, 1)] + [w[-1]],
            [b[2 * m + i] for m in mods for i in (0, 1)] + [b[-1]])
  rng = np.random.RandomState(1000 + depth)
  ws, bs = [], []
  for l in range(2 * depth):
    cin = 2 if l == 0 else 32
    gain = 1.0 if l % 2 == 0 else 0.5              # damped `_b` layers keep the residual stream O(1)
    ws.append((rng.randn(3, 3, 3, cin, 32) * gain * np.sqrt(2.0 / (27 * cin))).astype(np.float32))
    bs.append((rng.randn(32) * 0.1).astype(np.float32))
  ws.append((rng.randn(1, 1, 1, 32, 1) / np.sqrt(32.0)).astype(np.float32))
  bs.append((np.sign(rng.randn(1)) * 0.5).astype(np.float32))   # |b_lom| of the order of FIB-25's 0.31

  return ws, bs


def sweep_patches(fov, n):
  """n (seed, image) patches: phantom image crops and mixed seeds (pad value, +-logit(0.95), a few +-20)."""
  from ffn_b200.synthetic import voronoi_phantom
  fov = tuple(fov)
  vol = voronoi_phantom(tuple(s + 8 for s in fov), seed=sum(fov), cell_volume=4000.0)
  image = (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)
  rng = np.random.RandomState(int(np.prod(fov)) % 9973)
  seeds, imgs = [], []
  for _ in range(n):
    o = [int(rng.randint(0, 9)) for _ in range(3)]
    imgs.append(image[o[0]:o[0] + fov[0], o[1]:o[1] + fov[1], o[2]:o[2] + fov[2]])
    u = rng.rand(*fov)
    s = np.full(fov, PAD, np.float32)
    s[u < 0.45] = np.float32(INIT)
    s[(u >= 0.45) & (u < 0.6)] = np.float32(-INIT)
    s[u >= 0.995] = np.float32(20.0)
    s[(u >= 0.99) & (u < 0.995)] = np.float32(-20.0)
    s[tuple(f // 2 for f in fov)] = np.float32(INIT)
    seeds.append(s)
  return np.ascontiguousarray(seeds), np.ascontiguousarray(imgs)


# ------------------------------------------------------------------------------------------------------------------
# The conv stack in the device's row space (float64), with switchable bugs
# ------------------------------------------------------------------------------------------------------------------

def rowspace_logits(w, b, seed, image, x_mask=True, zero_line=True, residual=None, lom_bias_twice=False,
                    pad_twice=False):
  """Logits of one (Z, Y, X) patch, computed the way the kernels lay the FoV out: voxel (z, y, x) is row
  z*pp + y*fx + x with pp = (fy + 1)*fx (one zero line after every z-plane), a 3x3x3 tap is the row offset
  dz*pp + dy*fx + dx, rows outside the FoV read zero, and the dx = -1 / +1 taps are masked at x = 0 / fx - 1.

    x_mask=False      dx taps not masked: x = 0 reads the previous row (the end of the line above)
    zero_line=False   pp = fy*fx: a dy tap at y = 0 / fy - 1 reads the neighbouring z-plane
    residual='add'    depth 1: the last layer adds its input as if it were a residual
    residual='drop'   the first residual module leaves out its skip connection
    lom_bias_twice    conv_lom's bias added twice
    pad_twice         the pad value added once more to every pad-valued seed voxel
  """
  fz, fy, fx = seed.shape
  pp = (fy + 1) * fx if zero_line else fy * fx
  L = fz * pp
  reach = pp + fx + 1
  s = np.asarray(seed, np.float64)
  if pad_twice:
    s = np.where(np.asarray(seed) == np.float32(PAD), s + np.float64(np.float32(PAD)), s)
  x = np.arange(fx)
  m_up = np.tile(np.where(x == 0, 0.0, 1.0), fz * pp // fx) if x_mask else np.ones(L)
  m_dn = np.tile(np.where(x == fx - 1, 0.0, 1.0), fz * pp // fx) if x_mask else np.ones(L)
  valid = np.zeros((fz, pp // fx, fx), bool)
  valid[:, :fy, :] = True
  valid = torch.from_numpy(valid.reshape(L))
  m_up, m_dn = torch.from_numpy(m_up), torch.from_numpy(m_dn)

  def to_rows(v):                          # [C, Z, Y, X] -> [C, L]
    out = torch.zeros((v.shape[0], fz, pp // fx, fx), dtype=torch.float64)
    out[:, :, :fy, :] = v
    return out.reshape(v.shape[0], L)

  def conv(a, wk, bias):                   # a [Cin, L] -> [32, L]
    ap = torch.nn.functional.pad(a, (reach, reach))
    wt = torch.from_numpy(np.asarray(wk, np.float64))   # [3, 3, 3, Cin, Cout]
    acc = [torch.zeros((wt.shape[4], L), dtype=torch.float64) for _ in range(3)]
    for kz in range(3):
      for ky in range(3):
        for kx in range(3):
          o = (kz - 1) * pp + (ky - 1) * fx + (kx - 1)
          acc[kx] += wt[kz, ky, kx].T @ ap[:, reach + o:reach + o + L]
    out = acc[0] * m_up + acc[1] + acc[2] * m_dn + torch.from_numpy(np.asarray(bias, np.float64))[:, None]
    return torch.where(valid, out, torch.zeros((), dtype=torch.float64))   # pad rows are never written

  relu = torch.relu
  depth = (len(w) - 1) // 2
  net = to_rows(torch.from_numpy(np.stack([np.asarray(image, np.float64), s])))
  h = relu(conv(net, w[0], b[0]))
  net = conv(h, w[1], b[1])
  if residual == 'add' and depth == 1:
    net = net + h
  for m in range(1, depth):
    skip = net
    net = relu(conv(relu(net), w[2 * m], b[2 * m]))
    net = conv(net, w[2 * m + 1], b[2 * m + 1])
    if not (residual == 'drop' and m == 1):
      net = net + skip
  upd = torch.from_numpy(np.asarray(w[-1], np.float64).reshape(32)) @ relu(net) + float(b[-1][0])
  if lom_bias_twice:
    upd = upd + float(b[-1][0])
  upd = upd.reshape(fz, pp // fx, fx)[:, :fy, :].numpy()
  return s + upd


def _variants(depth):
  """name -> (kwargs, the bound the GPU test must exceed by 10x to catch it)."""
  out = {'x_unmasked': (dict(x_mask=False), TOL_FP16),
         'dy_across_planes': (dict(zero_line=False), TOL_FP16),
         'residual': (dict(residual='add' if depth == 1 else 'drop'), TOL_FP16),
         'pad_twice': (dict(pad_twice=True), TOL_FP16),
         # a constant offset of b_lom (0.31 for FIB-25): the fp16 check against the fp16-operand oracle catches it
         'lom_bias_twice': (dict(lom_bias_twice=True), TOL_FP16_OP)}
  return out


# ------------------------------------------------------------------------------------------------------------------
# Tests
# ------------------------------------------------------------------------------------------------------------------

def _check_canvas(canvas, g, p):
  np.testing.assert_array_equal(np.asarray(canvas.trace, dtype=np.int32).reshape(-1, 3), g[p + 'trace'])
  np.testing.assert_array_equal(canvas.segmentation, g[p + 'segmentation'])
  np.testing.assert_array_equal(canvas.seed, g[p + 'seed_canvas'])
  np.testing.assert_array_equal(canvas.seg_prob, g[p + 'seg_prob'])
  origins = np.array([(k,) + v[0] + (v[1],) for k, v in sorted(canvas.origins.items())], dtype=np.int64).reshape(-1, 5)
  np.testing.assert_array_equal(origins, g[p + 'origins'])
  owner, ids, cnt = [], [], []
  for k, v in sorted(canvas.overlaps.items()):
    for i, c in zip(v[0], v[1]):
      owner.append(k); ids.append(int(i)); cnt.append(int(c))
  np.testing.assert_array_equal(np.asarray([owner, ids, cnt], dtype=np.int64).reshape(3, -1),
                                g[p + 'overlaps'].reshape(3, -1))
  want = json.loads(str(g[p + 'counters']))
  for name in ('skip_threshold', 'skip_invalid_pos', 'voxels-segmented', 'voxels-overlapping',
               'inference-calls', 'seed_got_too_weak'):
    assert canvas.counters.get(name, 0) == want.get(name, 0), name
  assert canvas.counters['segment_at-calls'] == want['segment_at-loop-calls']


@pytest.mark.parametrize('name', ['g9', 'g5', 'g3'])
def test_toy_flood_fill_bit_exact_at_other_geometries(golden_dir, name):
  """fov (9, 17, 25) / deltas (2, 4, 6), fov (5, 33, 33) / deltas (0, 8, 8) and fov (3, 3, 3) / deltas (1, 1, 1):
  the oracle loop reproduces the reference's own segment_all bit for bit, including the seeds rejected by
  min_boundary_dist (-1 markers) and by min_segment_size."""
  g = _load(golden_dir, 'toy_geometry_flood_fill.npz')
  p = name + '_'
  fov, deltas = tuple(int(v) for v in g[p + 'fov']), tuple(int(v) for v in g[p + 'deltas'])
  opts = ff.Options(min_segment_size=int(g[p + 'min_segment_size']),
                    min_boundary_dist=tuple(int(v) for v in g[p + 'min_boundary_dist']))
  canvas = ff.Canvas(toy_net, toy_image(g[p + 'cells']), fov, deltas, opts)
  canvas.segment_all(g[p + 'seeds'])
  _check_canvas(canvas, g, p)
  n_small = json.loads(str(g[p + 'counters']))['segment_at-loop-calls'] - g[p + 'origins'].shape[0]
  assert n_small > 0 and (g[p + 'segmentation'] == -1).sum() > n_small   # both rejections occur
  assert g[p + 'origins'].shape[0] >= 2


def test_rowspace_stack_equals_the_network_oracle(golden_dir):
  """The row-space restatement without bugs is the conv stack (ConvStackOracle, float64), at an anisotropic FoV
  with fx = 3 (every x border is a tile-row border) and at depth 1 and 3."""
  from oracle.network import ConvStackOracle
  for fov, depth in (((5, 7, 3), 1), ((7, 5, 9), 3)):
    w, b = sweep_weights(golden_dir, depth, 'fib25')
    seeds, imgs = sweep_patches(fov, 1)
    want = seeds[0].astype(np.float64) + ConvStackOracle(w, b, dtype=torch.float64).update(seeds[0], imgs[0])
    got = rowspace_logits(w, b, seeds[0], imgs[0])
    assert np.abs(got - want).max() <= 1e-10 * max(1.0, np.abs(want).max()), (fov, depth)


def test_fp16_bounds_have_headroom_at_every_depth(golden_dir):
  """The fp16 bounds are not widened with depth: at every case of the sweep (depth 16 included), two correct
  fp16-operand implementations (fp32 and float64 accumulation) differ by at most half of TOL_FP16_OP, and the
  fp16-operand oracle is within half of TOL_FP16 of float64."""
  from oracle.network import ConvStackOracle
  for case, fov, depth, kind in SWEEP:
    w, b = sweep_weights(golden_dir, depth, kind)
    seeds, imgs = sweep_patches(fov, 1)
    a = ConvStackOracle(w, b, operand_round='fp16')(seeds, imgs)
    c = ConvStackOracle(w, b, operand_round='fp16', dtype=torch.float64)(seeds, imgs)
    d = ConvStackOracle(w, b, dtype=torch.float64)(seeds, imgs)
    assert np.abs(a - c).max() <= TOL_FP16_OP / 2, case
    assert np.abs(c - d).max() <= TOL_FP16 / 2, case


@pytest.mark.parametrize('case', [c[0] for c in SWEEP])
def test_tolerances_catch_one_tap_bugs(golden_dir, case):
  """Each deliberate bug moves some logit by >= 10x the bound the GPU test applies at this geometry and depth."""
  _, fov, depth, kind = next(c for c in SWEEP if c[0] == case)
  w, b = sweep_weights(golden_dir, depth, kind)
  seeds, imgs = sweep_patches(fov, 1)
  good = rowspace_logits(w, b, seeds[0], imgs[0])
  assert np.isfinite(good).all() and np.abs(good - seeds[0]).max() < 100.0     # activations stay O(1)
  report = {}
  for name, (kw, tol) in _variants(depth).items():
    diff = float(np.abs(rowspace_logits(w, b, seeds[0], imgs[0], **kw) - good).max())
    report[name] = round(diff, 4)
    assert diff >= 10 * tol, (case, name, diff, tol)
  print(case, report)
