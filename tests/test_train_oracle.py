"""The training-step oracle (oracle/train_step.py) on the CPU, the trainer's compiled kernels and its refusals."""

import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import train_cases
from oracle import exact_net, network, train_step as ts

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('depth', [1, 2])
def test_gradients_equal_central_differences(depth):
  w, b = train_cases.real_net(depth, depth)
  seed, image, labels, lw = train_cases.real_batch((5, 5, 5), 2, 3)
  _, _, gw, gb, loss = ts.gradients(w, b, seed, image, labels, lw)
  rng = np.random.RandomState(4)
  h = 1e-6
  for k in range(len(w)):
    for arr, grads in ((w, gw), (b, gb)):
      idx = tuple(rng.randint(s) for s in arr[k].shape)
      plus = [a.astype(np.float64).copy() for a in arr]
      minus = [a.astype(np.float64).copy() for a in arr]
      plus[k][idx] += h
      minus[k][idx] -= h
      lp = ts.gradients(*((plus, b) if arr is w else (w, plus)), seed, image, labels, lw)[4]
      lm = ts.gradients(*((minus, b) if arr is w else (w, minus)), seed, image, labels, lw)[4]
      fd = (lp - lm) / (2 * h)
      assert abs(fd - grads[k][idx]) <= 1e-6 * max(1.0, abs(fd)), (k, idx, fd, grads[k][idx])


def test_forward_logits_equal_the_network_oracle():
  w, b = train_cases.real_net(3, 7)
  seed, image, _, _ = train_cases.real_batch((7, 9, 5), 2, 8)
  got = ts.gradients(w, b, seed, image, dlogits=np.zeros(seed.shape))[0]
  want = network.ConvStackOracle(w, b, dtype=torch.float64).update(seed, image) + seed
  np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


def test_optimizer_formulas_by_hand():
  w, g = [np.float32([1.0, -2.0])], [np.float32([0.5, -3.0])]   # -3 is clipped to -0.7
  st = ts.OptState(w, 'sgd')
  w1 = ts.update(w, g, st, 0.25)
  np.testing.assert_array_equal(w1[0], np.float32([1 - 0.125, -2 + 0.175]))
  st = ts.OptState(w, 'momentum')
  w1 = ts.update(w, g, st, 0.5, momentum=0.5)
  w2 = ts.update(w1, g, st, 0.5, momentum=0.5)
  np.testing.assert_array_equal(w1[0], np.float32([0.75, -1.65]))              # a = g
  np.testing.assert_array_equal(w2[0], np.float32([0.75 - 0.375, -1.65 + 0.525]))  # a = 0.5 g + g
  st = ts.OptState(w, 'adam', beta1=0.5, beta2=0.75)
  w1 = ts.update(w, g, st, 0.125, beta1=0.5, beta2=0.75, epsilon=0.0)
  # t = 1: m = g / 2, v = g^2 / 4, alpha = lr sqrt(1 - 0.75) / (1 - 0.5) = lr: w -= lr sign(g)
  np.testing.assert_array_equal(w1[0], np.float32([1 - 0.125, -2 + 0.125]))
  w2 = ts.update(w1, g, st, 0.125, beta1=0.5, beta2=0.75, epsilon=0.0)
  # t = 2: m = 3 g / 4, v = 7 g^2 / 16, alpha = lr sqrt(1 - 9/16) / (3/4): step = lr (sqrt(7) / 3) (3/4) / (sqrt(7) / 4)
  np.testing.assert_allclose(w2[0], np.float32([1 - 0.25, -2 + 0.25]), rtol=0, atol=1e-6)
  assert st.beta1_power == np.float32(0.125) and st.beta2_power == np.float32(0.421875)


def test_bf16_rounding_is_round_to_nearest_even():
  x = np.array([1 + 2 ** -8, 1 + 3 * 2 ** -8, 1 + 2 ** -8 + 2 ** -20, -(1 + 2 ** -8), 2 ** -130])
  np.testing.assert_array_equal(ts.round_bf16(x), [1, 1 + 2 ** -6, 1 + 2 ** -7, -1, 2 ** -130])
  # the wrong modes of the bugs 'bf16_truncate' and 'bf16_half_away'
  np.testing.assert_array_equal(ts.round_bf16(x, 'rtz'), [1, 1 + 2 ** -7, 1, -1, 2 ** -130])
  np.testing.assert_array_equal(ts.round_bf16(x, 'rha'), [1 + 2 ** -7, 1 + 2 ** -6, 1 + 2 ** -7, -(1 + 2 ** -7),
                                                          2 ** -130])


def test_exact_case_satisfies_the_premise_and_large_sums_are_rejected():
  w, b, seed, image, labels, lw, dl = train_cases.exact_case((5, 7, 9), 2, 2)
  assert not ts.premise_violations(w, b, seed, image, dl)
  np.testing.assert_array_equal(ts.gradients(w, b, seed, image, dlogits=dl, bf16=True)[0], 0)
  big = [x * np.float32(2.0 ** 20) if i == 2 else x for i, x in enumerate(w)]
  names = [n for n, _, _ in ts.premise_violations(big, b, seed, image, dl)]
  assert 'conv2 forward' in names and any('wgrad' in n for n in names)


@pytest.mark.parametrize('name', sorted(train_cases.PROBE_BUGS))
def test_every_probe_satisfies_the_premise(name):
  w, b, seed, image, labels, lw, dl = train_cases.probe(name)
  assert not ts.premise_violations(w, b, seed, image, dl)
  assert np.count_nonzero(dl) > dl.size // 3


@pytest.mark.parametrize('bug', ts.BUGS)
def test_each_probe_bug_changes_a_gradient(bug):
  """The bugs the exact GPU tests catch though a tolerance would not, each on every probe listed for it: a ReLU
  derivative of 1 at a pre-activation of exactly 0, a residual gradient not carried past the skip, an input gradient
  without the tap flip, a wrong bf16 rounding mode, bias gradients of the rounded output gradient, a residual gradient
  rounded to bf16 and a rounded seed in the head.  Each changes the logits or a gradient."""
  names = [n for n, bugs in train_cases.PROBE_BUGS.items() if bug in bugs]
  assert names
  for name in names:
    w, b, seed, image, _, _, dl = train_cases.probe(name)
    rl, _, rw, rb, _ = ts.gradients(w, b, seed, image, dlogits=dl, bf16=True)
    bl, _, bw, bb, _ = ts.gradients(w, b, seed, image, dlogits=dl, bf16=True, bug=bug)
    assert any(not np.array_equal(x, y) for x, y in zip([rl] + rw + rb, [bl] + bw + bb)), name


def test_loss_gradient_at_logit_zero_is_one_half_minus_the_label():
  """At x = 0 the derivative is sigmoid(0) - z = 1/2 - z (autograd of TF's formula would take 1 - z there)."""
  w, b, seed, image, labels, lw, dl = train_cases.exact_case((3, 5, 7), 1, 2, density=0.5)
  logits, got, _, _, _ = ts.gradients(w, b, seed, image, labels, lw, bf16=True)
  np.testing.assert_array_equal(logits, 0)
  np.testing.assert_array_equal(got, dl)


def test_head_reference_equals_sigmoid_xent_and_autograd():
  w, b, seed, image, labels, lw = train_cases.head_grid_case()
  ref = ts.head_reference(seed, labels, lw)
  x = torch.from_numpy(seed.astype(np.float64)).requires_grad_()
  loss = ts.sigmoid_xent(x, labels, lw)
  loss.backward()
  assert abs(float(loss.detach()) - ref['loss']) <= 1e-12 * abs(ref['loss'])
  np.testing.assert_allclose(x.grad.numpy(), ref['dlogits'], rtol=1e-12, atol=0)
  # conv_lom's sums against the oracle's backward pass of the same step (w_lom = b_lom = 0: logits = seed)
  act = F.relu(ts.forward(*ts._params(w, b), seed, image, bf16=True)[1]).detach().numpy()
  ref = ts.head_reference(seed, labels, lw, act)
  _, _, gw, gb, _ = ts.gradients(w, b, seed, image, labels, lw, bf16=True)
  np.testing.assert_allclose(gw[-1].reshape(-1), ref['w_lom'], rtol=1e-12, atol=0)
  assert abs(gb[-1][0] - ref['b_lom']) <= 1e-12 * np.abs(ref['dlogits']).sum()


@pytest.mark.slow
def test_trainer_kernels_issue_bf16_wgmma_without_spills():
  """ptxas -v of train.cu with the library's own flags, and the SASS of the built library."""
  from ffn_b200 import build
  cuobjdump = os.path.join(os.path.dirname(build.nvcc_path()), 'cuobjdump')
  if not os.path.isabs(build.nvcc_path()) or not os.path.exists(cuobjdump):
    pytest.skip('nvcc / cuobjdump not found')
  with tempfile.TemporaryDirectory() as d:
    log = build.compile(os.path.join(build.CSRC, 'train.cu'), os.path.join(d, 'train.cubin'), ['-cubin', '-Xptxas', '-v'])
  sass = subprocess.run([cuobjdump, '-sass', build.build()], capture_output=True, text=True, check=True).stdout
  assert 'serialized' not in log, log
  props = re.findall(r'Function properties for (\w+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                     r'(\d+) bytes spill loads', log)
  assert len(props) >= 7, log
  for name, stack, stores, loads in props:
    assert (stack, stores, loads) == ('0', '0', '0'), name
  funcs = {f.split('\n', 1)[0].strip(): f for f in re.split(r'\n\s*Function : ', sass)[1:]}
  mma = [n for n in funcs if n.startswith('_ZN3trk') and ('4conv' in n or '5wgrad' in n)]
  assert len(mma) == 7, [n for n in funcs if n.startswith('_ZN3trk')]
  for n in mma:
    assert re.search(r'HGMMA\.64x32x16\.F32\.BF16', funcs[n]), n


def test_trainer_create_fails_loudly_without_gpu():
  if torch.cuda.is_available():
    pytest.skip('GPU present')
  from ffn_b200.training.trainer import Trainer
  w, b = exact_net.random_net(1, 0)
  with pytest.raises(RuntimeError, match='no CUDA device'):
    Trainer(w, b, (3, 3, 3))


def test_trainer_refuses_what_the_engine_refuses_and_unpinned_optimizers():
  from ffn_b200 import _lib
  from ffn_b200.training.trainer import Trainer
  w, b = exact_net.random_net(1, 0)
  for opt in ('adagrad', 'rmsprop'):
    with pytest.raises(ValueError, match='not supported'):
      Trainer(w, b, (3, 3, 3), optimizer=opt)
  lib = _lib.load()
  ptrs = lambda arrs: (C.c_void_p * len(arrs))(*[np.ascontiguousarray(a, np.float32).ctypes.data for a in arrs])
  td = _lib.TrainDesc(optimizer=0, max_batch=1)
  for fov, depth, feat in (((4, 3, 3), 1, 32), ((3, 3, 3), 0, 32), ((3, 3, 3), 17, 32), ((3, 3, 3), 1, 16)):
    desc = _lib.ModelDesc(fov_zyx=_lib.i3(fov), deltas_zyx=_lib.i3((0, 0, 0)), depth=depth, features=feat)
    h = C.c_void_p()
    assert lib.ffn_trainer_create(0, C.byref(desc), ptrs(w), ptrs(b), C.byref(td), C.byref(h)) != 0
    msg = lib.ffn_last_error()
    assert lib.ffn_engine_create(0, C.byref(desc), ptrs(w), ptrs(b), 0, C.byref(h)) != 0
    assert lib.ffn_last_error() == msg
