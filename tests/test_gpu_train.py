"""Training steps on the device against the float64 oracle (oracle/train_step.py).

Exactly representable steps (tests/train_cases.py) pin every weight and bias gradient bit for bit; real-valued FIB-25
steps are bounded through the bf16 unit roundoff; the update is pinned op by op; steps are deterministic, lower the
loss, and leave weights an Engine runs."""

import os

import numpy as np
import pytest

import train_cases
from oracle import train_step as ts

pytestmark = pytest.mark.gpu

U_BF16 = 2.0 ** -8   # unit roundoff of bf16 (8 significant bits)


def _trainer(w, b, fov, batch, **kw):
  from ffn_b200.training.trainer import Trainer
  return Trainer(w, b, fov, batch_size=batch, **kw)


# weighted: voxels with a non-zero loss weight, enough to reach every weight and few enough that every weight-gradient
# sum stays exact (deeper stacks spread each voxel's gradient over more rows, on a finer grid)
@pytest.mark.parametrize('fov,depth,batch,weighted', [((3, 3, 3), 1, 1, 800), ((9, 17, 25), 2, 3, 800),
                                                      ((17, 33, 33), 2, 4, 800), ((33, 33, 33), 12, 1, 60),
                                                      ((3, 3, 3), 2, 4, 800)])
def test_exact_gradients_equal_the_oracle(fov, depth, batch, weighted):
  density = min(1.0, weighted / (batch * int(np.prod(fov))))
  w, b, seed, image, labels, lw, dl = train_cases.exact_case(fov, depth, batch, density=density)
  tr = _trainer(w, b, fov, batch)
  got_dl, gw, gb, _ = tr.gradients(seed, image, labels, lw)
  tr.close()
  np.testing.assert_array_equal(got_dl, dl)        # every logit is exactly 0
  assert not ts.premise_violations(w, b, seed, image, got_dl)
  _, _, rw, rb, _ = ts.gradients(w, b, seed, image, bf16=True, dlogits=got_dl)
  assert any(np.abs(g).max() > 0 for g in rw[:-1])
  for i, (g, r) in enumerate(zip(gw, rw)):
    np.testing.assert_array_equal(g, r.astype(np.float32).reshape(g.shape), err_msg='weights %d' % i)
  for i, (g, r) in enumerate(zip(gb, rb)):
    np.testing.assert_array_equal(g, r.astype(np.float32).reshape(g.shape), err_msg='biases %d' % i)


def test_a_smaller_batch_after_a_larger_one_gives_the_gradients_of_a_fresh_trainer():
  # (9, 17, 25): the rows past two patches, up to the 1 024-row split, reach past the third patch's padding
  w, b, seed, image, labels, lw, _ = train_cases.exact_case((9, 17, 25), 2, 3, density=0.5)
  used = _trainer(w, b, (9, 17, 25), 3)
  used.gradients(seed, image, labels, lw)
  got = used.gradients(seed[:2], image[:2], labels[:2], lw[:2])
  used.close()
  fresh = _trainer(w, b, (9, 17, 25), 3)
  want = fresh.gradients(seed[:2], image[:2], labels[:2], lw[:2])
  fresh.close()
  for x, y in zip([got[0]] + got[1] + got[2], [want[0]] + want[1] + want[2]):
    np.testing.assert_array_equal(x, y)
  assert got[3] == want[3]


@pytest.fixture(scope='module')
def fib25_batch(golden_dir):
  from ffn_b200 import synthetic, tf_checkpoint
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))
  vol, cells = synthetic.voronoi_phantom((80, 80, 80), seed=5, return_cells=True)
  image = ((vol.astype(np.float32) - np.float32(128)) / np.float32(33)).astype(np.float32)
  rng = np.random.RandomState(1)
  crops, labs, seeds = [], [], []
  for _ in range(2):
    z, y, x = rng.randint(0, 80 - 33, 3)
    crops.append(image[z:z + 33, y:y + 33, x:x + 33])
    c = cells[z:z + 33, y:y + 33, x:x + 33]
    lab = (c == c[16, 16, 16]).astype(np.float32)
    labs.append(np.float32(0.05) + np.float32(0.9) * lab)      # soft labels
    s = np.full((33, 33, 33), -0.4, np.float32)
    s[16, 16, 16] = 0.95
    seeds.append(s)
  return w, b, np.stack(seeds), np.stack(crops), np.stack(labs)


def _rel(a, b):
  return float(np.linalg.norm(np.ravel(a) - np.ravel(b)) / max(np.linalg.norm(np.ravel(b)), 1e-30))


def test_real_valued_gradients_within_bf16_bounds(fib25_batch):
  w, b, seed, image, labels = fib25_batch
  tr = _trainer(w, b, (33, 33, 33), 2)
  dl, gw, gb, loss = tr.gradients(seed, image, labels)
  tr.close()
  nconv = len(w) - 1
  # Against the bf16-operand oracle the device rounds the same values; only fp32 accumulation order differs, which
  # moves a rounded operand by one bf16 ulp (2u) only where a value sits within ~2^-24 of a rounding boundary.
  # Normwise the difference stays below one unit roundoff u.  Against the pure float64 oracle, a gradient carries the
  # roundings of two operands per conv in the forward pass (input and weights) and, in the backward pass, of the output
  # gradient of every conv above it: at most 2 (2 nconv + 1) roundings of relative size <= u each.  They are
  # independent, so normwise they add in quadrature: sqrt(2 (2 nconv + 1)) u (0.039 at depth 12).  Measured on an
  # H100: 0.0033 against the bf16 oracle, 0.017 against the float64 one.
  for bf16, bound in ((True, U_BF16), (False, np.sqrt(2 * (2 * nconv + 1)) * U_BF16)):
    _, rdl, rw, rb, rloss = ts.gradients(w, b, seed, image, labels, bf16=bf16)
    print('bf16' if bf16 else 'f64', 'loss', loss, rloss, 'dlogits', _rel(dl, rdl),
          'weights', max(_rel(g, r) for g, r in zip(gw, rw)), 'biases', max(_rel(g, r) for g, r in zip(gb, rb)))
    assert abs(loss - rloss) <= bound * abs(rloss)
    assert _rel(dl, rdl) <= bound
    for g, r in zip(gw + gb, rw + rb):
      assert _rel(g, r) <= bound


@pytest.mark.parametrize('optimizer', ['sgd', 'momentum', 'adam'])
def test_update_is_the_oracle_update_of_the_clipped_gradients(fib25_batch, optimizer):
  w, b, seed, image, labels = fib25_batch
  lw = np.full(labels.shape, 3e5, np.float32)      # gradient entries far beyond +-0.7
  tr = _trainer(w, b, (33, 33, 33), 2, optimizer=optimizer, learning_rate=0.01)
  state = ts.OptState(w + b, optimizer)
  beyond = 0
  for _ in range(2):
    ws, bs = tr.weights()
    _, gw, gb, _ = tr.gradients(seed, image, labels, lw)
    beyond += sum(int((np.abs(g) > 0.7).sum()) for g in gw + gb)
    want = ts.update(ws + bs, gw + gb, state, np.float32(0.01))
    tr.step(seed, image, labels, lw)
    nw, nb = tr.weights()
    for i, (g, r) in enumerate(zip(nw + nb, want)):
      np.testing.assert_array_equal(g, r, err_msg='%s parameter %d' % (optimizer, i))
  assert tr.global_step == 2
  assert beyond > 0
  tr.close()


def test_identical_steps_give_identical_weights(fib25_batch):
  w, b, seed, image, labels = fib25_batch
  out = []
  for _ in range(2):
    tr = _trainer(w, b, (33, 33, 33), 2, optimizer='adam')
    for k in range(5):
      tr.step(np.roll(seed, k, 1), image, labels)
    out.append(tr.weights())
    tr.close()
  for x, y in zip(out[0][0] + out[0][1], out[1][0] + out[1][1]):
    np.testing.assert_array_equal(x, y)


def test_repeated_steps_lower_the_loss(fib25_batch):
  w, b, seed, image, labels = fib25_batch
  tr = _trainer(w, b, (33, 33, 33), 2, learning_rate=0.002)
  losses = [tr.step(seed, image, labels)[1] for _ in range(6)]
  tr.close()
  print('losses', losses)
  assert all(b < a for a, b in zip(losses, losses[1:])), losses


def test_trained_weights_run_in_an_engine(fib25_batch):
  from ffn_b200 import _lib, engine as eng
  w, b, seed, image, labels = fib25_batch
  tr = _trainer(w, b, (33, 33, 33), 2, optimizer='momentum', learning_rate=0.01)
  for _ in range(3):
    tr.step(seed, image, labels)
  ws, bs = tr.weights()
  logits, _ = tr.step(seed, image, labels)         # the forward pass of the weights read above
  tr.close()
  e = eng.Engine(ws, bs, (33, 33, 33), (8, 8, 8), compute_mode=_lib.COMPUTE_FP16_TC)
  got = e.predict(seed, image)
  e.close()
  # The bound tests/test_gpu_parity.py holds the fp16 engine to against fp32 logits (measured here: 0.024 between the
  # fp16 engine and the bf16 trainer).  A weight in the wrong layout moves logits by far more.
  err = float(np.abs(got - logits).max())
  print('engine vs trainer logits', err)
  assert err <= 4e-2


def test_trainers_return_their_device_memory(fib25_batch):
  from test_gpu_lifetime import _process_device_memory
  w, b, seed, image, labels = fib25_batch
  memory = []
  for _ in range(6):
    tr = _trainer(w, b, (33, 33, 33), 2)
    tr.step(seed, image, labels)
    tr.close()
    memory.append(_process_device_memory())
  print('device memory after each trainer (bytes, NVML):', memory)
  if any(m is None for m in memory):
    pytest.skip('NVML lists no compute process for this pid: memory not checked')
  assert memory[-1] <= memory[0], memory
