"""The tracker oracle against the reference's own EvalTracker (tests/golden/tracker_ref.npz): counters at every step,
summaries by tag at every summary point, images pixel for pixel outside their text, and each deliberate bug caught.
CPU only."""

import io
import math
import os

import numpy as np
import pytest

import examples_oracle as eo
import tracker_oracle as to
from ffn_b200.training import tracker as tk

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'tracker_ref.npz')
U = 2.0**-24   # float32 unit roundoff


def loss_bound(o, n_patches, n_voxels):
  """How far the fixture's float32 loss may lie from the oracle's float64 one.  Per voxel, the reference's float32
  max(x, 0) - x z + log1p(exp(-|x|)) makes at most 12 u |m| of error, m = max(x, 0) + |x z| + log1p(exp(-|x|)):
  u |x z| for the product, u (max + |x z|) for the difference, 4 u L each for exp and log1p (numpy's float32 libm,
  the exp error passing into log1p no more than that), u L and u |term| for the sum.  numpy's float32 mean sums
  pairwise (8 accumulators over blocks of 128: 16 sequential adds, 3 to combine, log2(N / 128) levels), so the
  mean adds (20 + log2 N) u of the sum of terms, which m bounds, and u for the division.  The loss variable then adds
  the patch means in float32: u times the running sum per patch, at most n_patches u of the sum.  Summed over
  patches with o.loss_mag = sum of mean(m)."""
  per_patch = 12 + 20 + math.ceil(math.log2(max(n_voxels, 2))) + 1
  return U * (per_patch + n_patches) * o.loss_mag + 1e-12


def run_case(i, c, bugs=(), ref=None, check=True):
  """Runs the oracle over the fixture's steps; with check, asserts every comparison; else returns whether any
  differs."""
  o = to.make(c, bugs)
  coords = eo.as_coords(c['rows'])
  rng = np.random.RandomState(c['logit_seed'])
  names = ['vol%d' % k for k in range(len(c['volumes']))]
  p = 'c%d/' % i
  pos = 0
  try:
    for step in range(eo.N_STEPS):
      pos += o.next(coords[pos:])[5]
      o.update(to.step_logits(rng, c))
      msg = '%s at step %d' % (c['tag'], step)
      moves_all = sum(o.moves_r.values())
      np.testing.assert_array_equal(moves_all, ref[p + 'moves'][step], err_msg=msg)
      for r, m in o.moves_r.items():
        assert p + 'moves_r=%d' % r in ref.files, msg + ': radius %d is not one of the reference\'s' % r
        np.testing.assert_array_equal(m, ref[p + 'moves_r=%d' % r][step], err_msg=msg)
      np.testing.assert_array_equal(o.pred, ref[p + 'prediction_counts'][step], err_msg=msg)
      assert [o.eval_voxels, 0] == ref[p + 'num_voxels'][step].tolist(), msg
      assert o.patches == ref[p + 'num_patches'][step][0], msg
      fov = o.steps * o.batch * int(np.prod(o.fov))
      assert ref[p + 'fov_stats'][step].tolist() == [fov, 0, fov], msg
      n_vox = int(np.prod(o.eval))
      assert abs(o.loss - float(ref[p + 'loss'][step][0])) <= loss_bound(o, o.patches, n_vox), msg
      if (step + 1) % to.SUMMARY_EVERY:
        continue
      bound = loss_bound(o, o.patches, n_vox) / max(o.patches, 1)
      state = o.state(reset=True)
      got = tk.summaries(state, names)
      s = p + 's%d/' % step
      want = dict(zip(ref[s + 'tags'].tolist(), ref[s + 'values'].tolist()))
      scalars = {t: v for t, v in got if not isinstance(v, tk.Image)}
      assert sorted(scalars) == sorted(want), msg
      for t, v in scalars.items():
        if t == 'eval/patch_loss':
          assert abs(v - want[t]) <= bound + U * abs(want[t]), (msg, t, v, want[t])
        else:
          assert v == want[t], (msg, t, v, want[t])
      if step == to.SUMMARY_EVERY - 1:
        images = {t: v for t, v in got if isinstance(v, tk.Image)}
        assert sorted(images) == sorted(f[len(s):] for f in ref.files if f.startswith(s + 'final_')), msg
        for t, v in images.items():
          k = int(t.split('/')[1])
          compare_image(v, ref[s + t], state.coords[k], names, msg + ' ' + t)
  except AssertionError:
    if check:
      raise
    return True
  return False


def compare_image(img, want, coord, names, msg):
  import PIL.Image
  import PIL.ImageDraw
  import PIL.ImageFont
  got = np.asarray(PIL.Image.open(io.BytesIO(img.png)).convert('RGB'))
  assert got.shape == want.shape == (img.height, img.width, 3), msg
  vol, (x, y, z) = coord
  im = PIL.Image.new('RGB', (img.width, img.height))
  box = PIL.ImageDraw.Draw(im).textbbox((1, 1), '%d,%d,%d\n%s' % (x, y, z, names[vol]),
                                        font=PIL.ImageFont.load_default())
  outside = np.ones(got.shape[:2], bool)
  outside[box[1]:box[3], box[0]:box[2]] = False
  np.testing.assert_array_equal(got[outside], want[outside], err_msg=msg)


@pytest.mark.parametrize('i', range(len(to.cases())))
def test_oracle_equals_reference(i):
  ref = np.load(GOLDEN)
  assert ref['n_cases'] == len(to.cases())
  run_case(i, eo.case_setup(to.cases()[i]), ref=ref)


@pytest.mark.parametrize('bug', to.BUGS)
def test_every_bug_changes_the_fixture(bug):
  ref = np.load(GOLDEN)
  assert any(run_case(i, eo.case_setup(case), (bug,), ref, check=False) for i, case in enumerate(to.cases())), bug


def test_cases_cover_every_move_type_and_prediction():
  """Across the cases: every move type at every radius a policy records moves at, all four prediction counts, centre
  moves of background examples (spurious at radius 0 under fixed, where only the centre and shifts of radius > 0 are
  recorded), and both sides of the eval threshold at its float32 neighbours."""
  ref = np.load(GOLDEN)
  by_r, pred = {}, np.zeros(4, np.int64)
  for i, case in enumerate(to.cases()):
    p = 'c%d/' % i
    rows = slice(to.SUMMARY_EVERY - 1, None, to.SUMMARY_EVERY)   # the counts just before each reset
    for k in ref.files:
      # max_pred_moves records at radius 0 only: its other radii (from model.shifts) stay empty
      if k.startswith(p + 'moves_r=') and (case[3] == 'fixed' or k.endswith('=0')):
        r = int(k.split('=')[1])
        by_r[r] = by_r.get(r, 0) + ref[k][rows].sum(0)
    pred += ref[p + 'prediction_counts'][rows].sum(0)
  assert len(by_r) >= 4
  for r, m in by_r.items():
    assert (m > 0).all(), (r, m)
  assert (pred > 0).all(), pred
  fixed = [i for i, c in enumerate(to.cases()) if c[3] == 'fixed']
  assert any(ref['c%d/moves_r=0' % i][-1][2] > 0 for i in fixed)
  snap = [i for i, c in enumerate(to.cases()) if c[-1] == 'eval']
  assert all(ref['c%d/prediction_counts' % i][-1][[0, 2]].min() > 0 for i in snap)


def test_radii_truncate():
  assert tk.radii([(8, 8, 8), (0, 8, 8), (0, 0, 8)]) == [0, 8, 11, 13]
  assert tk.radii([(2, 2, 2), (0, 2, 2), (2, 0, 0)]) == [0, 2, 3]
  assert tk.move_radius((0, 2, 2)) == 2   # 2.83: truncated, where rounding gives 3
