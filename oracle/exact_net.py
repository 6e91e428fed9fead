"""Exactly representable networks: conv stacks whose logits every correct implementation computes bit for bit.

Test infrastructure (see oracle/__init__.py), CPU only.  The conv stack of ConvStack3DFFNModel is restated in
float64 (`logits`), with the fp16 operand rounding of the tensor-core mode as an option and a switch per
deliberate arithmetic bug.  A network and its inputs satisfy the *premise* (`assert_exact`) when

* every weight, bias, image and seed value is dyadic, the 3x3x3 weights and every conv operand are exactly
  representable in fp16 (in the fp16 mode after the kernel's round-to-nearest-even, which the oracle applies too),
  and |w| * 2^10 <= 65504, so that the split-fp16 mode's pre-scaled weights have no lo part and every operand's lo
  part a - fp16(a) is itself an fp16 number;
* for every output of every convolution, with products on the grid 2^-q, sum |w| |a| + |bias| + |residual| < 2^(24-q)
  (and the same for conv_lom and for seed + update).  Then every partial sum, in any order, is a multiple of 2^-q
  below 2^(24-q): exact in fp32, and no alignment that keeps a 24-bit window can drop a bit.

Under the premise the fp32 and split-fp16 modes equal the float64 oracle, and the fp16 mode equals the float64
fp16-operand oracle, with no tolerance.  The probe networks (`PROBES`) put single values where a subtly wrong
kernel differs: fp32-only values in the residual stream, biases and seeds, conv outputs at fp16 rounding ties,
fp16 subnormal operands, ReLU at zero and the order of seed + b_lom + <relu(net), w_lom>.  `flood_net` is a
network under which the flood fill grows objects in bright cells with exactly representable logits.
"""

from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

FEAT = 32
F16_MAX = 65504.0
SPLIT_SHIFT = 10            # the split-fp16 mode packs w * 2^10 = hi + lo

# Bugs `logits` can apply, one at a time (the CPU tests show each one changes a logit of its probe):
BUGS = ('residual_fp16',      # the fp32 residual stream stored as fp16
        'bias_fp16',          # biases (b_lom included) rounded to fp16
        'seed_unrounded',     # fp16 mode: the seed operand of conv0_a not rounded to fp16
        'round_toward_zero',  # fp16 mode: the epilogue's fp16 conversion truncates
        'round_half_away',    # fp16 mode: ties rounded away from zero
        'flush_subnormal',    # fp16 operands (split mode: hi parts) below 2^-14 flushed to zero
        'bias_wrong_channel', # every layer's bias added to the next channel
        'lom_bias_twice',     # b_lom added twice
        'seed_plus_bias_first',  # fp32 (seed + b_lom) + <relu(net), w_lom> instead of seed + (b_lom + <.,.>)
        'no_relu_before_lom')    # conv_lom reads net instead of relu(net)


# ------------------------------------------------------------------------------------------------------------------
# fp16 rounding in float64
# ------------------------------------------------------------------------------------------------------------------

def round_f16(x, mode='rne', flush=False):
  """float64 values rounded to fp16 (to nearest even, toward zero or half away from zero), as float64."""
  x = np.asarray(x, np.float64)
  r = x.astype(np.float16)
  if mode != 'rne':
    r64 = r.astype(np.float64)
    toward0 = np.where(np.abs(r64) > np.abs(x), np.nextafter(r, np.float16(0)), r)
    if mode == 'rtz':
      r = toward0
    else:           # 'rha': at an exact tie take the neighbour away from zero
      t64 = toward0.astype(np.float64)
      away = np.nextafter(toward0, np.copysign(np.float16(np.inf), x).astype(np.float16)).astype(np.float64)
      tie = (t64 != x) & (x - t64 == away - x)
      r = np.where(tie, away, t64).astype(np.float16)
  out = r.astype(np.float64)
  if flush:
    out = np.where(np.abs(out) < 2.0 ** -14, 0.0, out)
  return out


def frac_bits(x):
  """Smallest k such that every value of x is a multiple of 2^-k (x finite)."""
  x = np.abs(np.asarray(x, np.float64)).ravel()
  x = x[x != 0]
  if x.size == 0:
    return 0
  _, e = np.frexp(x)                       # x = m * 2^e, 0.5 <= m < 1
  m = x * np.exp2(53 - e)                  # integer significand of 53 bits
  tz = np.zeros(x.shape, np.int64)
  mi = m.astype(np.uint64)
  for s in (32, 16, 8, 4, 2, 1):
    z = (mi & np.uint64((1 << s) - 1)) == 0
    tz += np.where(z, s, 0)
    mi = np.where(z, mi >> np.uint64(s), mi)
  return int(max(0, (53 - e - tz).max()))


def is_f16(x):
  x = np.asarray(x, np.float64)
  return bool(np.all(x.astype(np.float16).astype(np.float64) == x))


def is_f32(x):
  x = np.asarray(x, np.float64)
  return bool(np.all(x.astype(np.float32).astype(np.float64) == x))


# ------------------------------------------------------------------------------------------------------------------
# The float64 conv stack, with the fp16 operand rounding and the bugs
# ------------------------------------------------------------------------------------------------------------------

def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a, np.float64))


def _forward(w, b, seed, image, mode, bug, check):
  """Logits of a (B, Z, Y, X) or (Z, Y, X) batch in float64.  mode 'fp16' rounds every 3x3x3 conv operand to fp16
  (the tensor-core mode); 'fp32' and 'x2' do not.  `check(kind, operand, weight, bias, residual, out)` sees every
  convolution (operand after rounding; bias / residual broadcast to the output; None where absent)."""
  assert bug is None or bug in BUGS, bug
  seed = np.asarray(seed, np.float64)
  image = np.asarray(image, np.float64)
  batched = seed.ndim == 4
  if not batched:
    seed, image = seed[None], image[None]
  depth = (len(w) - 1) // 2
  fp16 = mode == 'fp16'
  rmode = {'round_toward_zero': 'rtz', 'round_half_away': 'rha'}.get(bug, 'rne')
  flush = bug == 'flush_subnormal'

  def rnd(x):                                # the operand a 3x3x3 conv reads
    if fp16:
      return _t(round_f16(x.numpy(), rmode, flush))
    if flush:                                # the split mode's hi parts flushed: the value is lost
      return torch.where(x.abs() < 2.0 ** -14, torch.zeros((), dtype=torch.float64), x)
    return x

  def bias(i):
    bb = np.asarray(b[i], np.float64).reshape(-1)
    if bug == 'bias_fp16':
      bb = round_f16(bb)
    if bug == 'bias_wrong_channel' and i < len(w) - 1:
      bb = np.roll(bb, 1)
    return _t(bb)

  def conv(x, i, res=None):
    wt = _t(np.asarray(w[i], np.float64)).permute(4, 3, 0, 1, 2).contiguous()
    y = F.conv3d(x, wt, None, padding=1)
    bb = bias(i)[None, :, None, None, None].expand_as(y)
    out = y + bb if res is None else y + bb + res
    if check is not None:
      check('conv', x, wt, bb, res, out)
    return out

  x0 = torch.stack([rnd(_t(image)), _t(seed) if bug == 'seed_unrounded' else rnd(_t(seed))], dim=1)
  net = conv(x0, 0).relu()
  net = conv(rnd(net), 1)
  if bug == 'residual_fp16':
    net = _t(round_f16(net.numpy()))
  for m in range(1, depth):
    skip = net
    h = conv(rnd(net.relu()), 2 * m).relu()
    net = conv(rnd(h), 2 * m + 1, skip)
    if bug == 'residual_fp16':
      net = _t(round_f16(net.numpy()))
  a = net if bug == 'no_relu_before_lom' else net.relu()
  wl = _t(np.asarray(w[-1], np.float64).reshape(FEAT))
  bl = float(bias(len(w) - 1)[0])
  dot = torch.einsum('bczyx,c->bzyx', a, wl)
  if check is not None:
    check('lom', a, wl, bl, None, dot + bl)
  upd = dot + bl
  if bug == 'lom_bias_twice':
    upd = upd + bl
  s = _t(seed)
  if bug == 'seed_plus_bias_first':
    out = ((s.numpy().astype(np.float32) + np.float32(bl)) + dot.numpy().astype(np.float32)).astype(np.float64)
  else:
    out = (s + upd).numpy()
    if check is not None:
      check('logit', s, None, upd, None, _t(out))
  out = out.astype(np.float32)
  return out if batched else out[0]


def logits(w, b, seed, image, mode='fp32', bug=None):
  """float64 logits rounded once to float32: the oracle of the fp32 / split-fp16 modes ('fp32', 'x2') and, with
  mode='fp16', the fp16-operand oracle of the tensor-core mode."""
  return _forward(w, b, seed, image, mode, bug, None)


def logits_f32(w, b, seed, image, mode='fp32'):
  """The same stack evaluated in float32 by torch's CPU conv3d (ConvStackOracle): under the premise it equals
  `logits` bit for bit, whatever order the CPU kernel sums in."""
  from oracle.network import ConvStackOracle
  return ConvStackOracle(w, b, operand_round='fp16' if mode == 'fp16' else None)(seed, image)


# ------------------------------------------------------------------------------------------------------------------
# The premise
# ------------------------------------------------------------------------------------------------------------------

class PremiseError(AssertionError):
  pass


def premise_margin(w, b, seeds, images, mode):
  """Checks the premise layer by layer and returns min over every sum of 2^(24-q) / (sum |terms|) (> 1)."""
  worst = [np.inf]
  for i, wi in enumerate(w):
    wi = np.asarray(wi, np.float64)
    if not (is_f32(wi) and is_f32(b[i])):
      raise PremiseError('layer %d: weights or biases not fp32' % i)
    if i < len(w) - 1:
      if not is_f16(wi):
        raise PremiseError('layer %d: weights not fp16-exact' % i)
      if np.abs(wi).max() * 2 ** SPLIT_SHIFT > F16_MAX:
        raise PremiseError('layer %d: |w| * 2^10 above the fp16 range' % i)
  for name, v in (('seed', seeds), ('image', images)):
    if not is_f32(v) or not np.isfinite(np.asarray(v, np.float64)).all():
      raise PremiseError('%s values not finite fp32' % name)

  def check(kind, x, wt, bias, res, out):
    xa = x.numpy()
    if kind == 'conv':
      if np.abs(xa).max() > F16_MAX:
        raise PremiseError('conv operand above the fp16 range')
      if mode == 'fp16' and not is_f16(xa):
        raise PremiseError('fp16 operand not rounded')
      if mode in ('fp32', 'x2'):
        lo = xa - round_f16(xa)
        if not is_f16(lo):
          raise PremiseError('operand lo part a - fp16(a) not fp16-exact')
        if mode == 'fp32' and not is_f32(xa):
          raise PremiseError('operand not fp32')
      wa = wt.numpy()
      q = frac_bits(xa) + frac_bits(wa)
      terms = [bias.numpy()] + ([] if res is None else [res.numpy()])
      q = max([q] + [frac_bits(t) for t in terms])
      tot = F.conv3d(x.abs(), wt.abs(), None, padding=1).numpy()
      for t in terms:
        tot = tot + np.abs(t)
    elif kind == 'lom':
      xa = x.numpy()
      wa = wt.numpy()
      q = max(frac_bits(xa) + frac_bits(wa), frac_bits(bias))
      tot = np.einsum('bczyx,c->bzyx', np.abs(xa), np.abs(wa)) + abs(bias)
    else:          # logit = seed + update, one fp32 add: the result and the update must be fp32
      if not (is_f32(bias.numpy()) and is_f32(out.numpy())):
        raise PremiseError('seed + update not exact in fp32')
      return
    if not (is_f32(out.numpy())):
      raise PremiseError('%s output not fp32' % kind)
    m = tot.max()
    lim = 2.0 ** (24 - q)
    if m >= lim:
      raise PremiseError('%s: sum |w||a| = %g >= 2^(24-%d)' % (kind, m, q))
    worst[0] = min(worst[0], lim / m if m > 0 else np.inf)

  _forward(w, b, seeds, images, mode, None, check)
  return worst[0]


def assert_exact(w, b, seeds, images, mode):
  """Raises PremiseError unless the network and these inputs satisfy the premise in `mode` ('fp16', 'x2', 'fp32')."""
  premise_margin(w, b, seeds, images, mode)


# ------------------------------------------------------------------------------------------------------------------
# Random sparse dyadic networks
# ------------------------------------------------------------------------------------------------------------------

def random_net(depth, seed):
  """A random sparse dyadic network of `depth` modules: each output channel of each 3x3x3 conv sums one or two taps
  with weights in {+-1/2, +-1, +-2}, biases are multiples of 1/8 in [-1/2, 1/2], conv_lom reads eight channels with
  weights +-1/2 and b_lom is a multiple of 1/4.  Halves appear only in every fourth conv (and there a +-2 tap comes
  with a +-1/2 one), so the activations gain at most one fractional bit per four layers and stay far below the
  bound at depth 16."""
  rng = np.random.RandomState(seed)
  ws, bs = [], []
  for l in range(2 * depth):
    cin = 2 if l == 0 else FEAT
    w = np.zeros((3, 3, 3, cin, FEAT), np.float32)
    for co in range(FEAT):
      k = rng.randint(3)
      if l % 4 == 0:
        pairs = [(1.0,), (0.5, 0.5), (2.0, 0.5)][k]
      elif l % 2 == 0:
        pairs = [(1.0,), (1.0,), (2.0,)][k]
      else:                                  # "_b": one +-1 tap
        pairs = (1.0,)
      for mag in pairs:
        tz, ty, tx = rng.randint(3, size=3)
        w[tz, ty, tx, rng.randint(cin), co] += np.float32(mag * rng.choice((-1.0, 1.0)))
    ws.append(w)
    bs.append((rng.randint(-4, 5, FEAT) / 8.0).astype(np.float32))
  wl = np.zeros(FEAT, np.float32)
  wl[rng.choice(FEAT, 8, replace=False)] = rng.choice((-0.5, 0.5), 8)
  ws.append(wl.reshape(1, 1, 1, FEAT, 1))
  bs.append(np.asarray([rng.randint(-4, 5) / 4.0], np.float32))
  return ws, bs


def random_patches(fov, n, seed):
  """n (seed, image) patches of dyadic values: images are multiples of 1/16 in [-4, 4), seeds a mix of the
  flood fill's pad and init values (-3, 2) and small multiples of 1/4."""
  rng = np.random.RandomState(seed)
  fov = tuple(int(f) for f in fov)
  imgs = (rng.randint(-64, 64, (n,) + fov) / 16.0).astype(np.float32)
  u = rng.rand(n, *fov)
  seeds = np.where(u < 0.5, -3.0, np.where(u < 0.8, 2.0, rng.randint(-16, 17, (n,) + fov) / 4.0)).astype(np.float32)
  return seeds, imgs


# ------------------------------------------------------------------------------------------------------------------
# Probe networks
# ------------------------------------------------------------------------------------------------------------------

def _zeros(depth):
  w = [np.zeros((3, 3, 3, 2 if l == 0 else FEAT, FEAT), np.float32) for l in range(2 * depth)]
  w.append(np.zeros((1, 1, 1, FEAT, 1), np.float32))
  b = [np.zeros(FEAT, np.float32) for _ in range(2 * depth)] + [np.zeros(1, np.float32)]
  return w, b


def _pass(w, layer, ci, co, v=1.0):
  w[layer][1, 1, 1, ci, co] = np.float32(v)


def probe_residual(fov):
  """conv0_b sums 1000 and 1/4 into the residual stream: 1000.25 is fp32 but not fp16.  The residual modules add
  nothing to that channel, so conv_lom reads 1000.25 only if the stream stays fp32.  The `_a` convs of the modules
  read the fp16-rounded value (1000.0) and pass it to another channel, which conv_lom weighs by -1."""
  w, b = _zeros(2)
  _pass(w, 0, 0, 0)                          # relu(image) (1000 at the patch's bright voxels)
  b[0][1] = 0.25                             # a constant 1/4
  _pass(w, 1, 0, 0)
  _pass(w, 1, 1, 0)                          # net0 = image + 1/4 = 1000.25
  _pass(w, 2, 0, 1)                          # module 1 _a: relu(net0) as an fp16 operand
  _pass(w, 3, 1, 1, -1.0)                    # module 1 _b: net1 = -fp16(net0) (+ 0 skip)
  w[-1][0, 0, 0, 0, 0] = 1.0
  w[-1][0, 0, 0, 1, 0] = -1.0                # update = 1000.25 + relu(-fp16(1000.25)) = 1000.25 (ReLU zeroes the other)
  b[-1][0] = 0.5
  seeds = np.full(fov, 2.0, np.float32)[None]
  imgs = np.where(np.indices(fov).sum(0) % 2 == 0, 1000.0, 0.0).astype(np.float32)[None]
  return w, b, seeds, imgs


def probe_bias(fov):
  """Biases that are fp32 but not fp16: 1 + 2^-12 on conv0_b, -1/3 to 2^-12 on a residual module's _b, and b_lom =
  2^-13 + 1/2."""
  w, b = _zeros(2)
  _pass(w, 0, 0, 0)
  _pass(w, 1, 0, 0)
  b[1][0] = 1.0 + 2.0 ** -12
  b[3][0] = 2.0 ** -11 + 2.0 ** -12 - 0.5
  w[-1][0, 0, 0, 0, 0] = 1.0
  b[-1][0] = 0.5 + 2.0 ** -13
  seeds = np.full(fov, -3.0, np.float32)[None]
  imgs = np.zeros(fov, np.float32)[None]
  imgs[0].reshape(-1)[::3] = 2.0
  return w, b, seeds, imgs


def probe_seed(fov):
  """Seeds that are fp32 but not fp16 (1000.25, 1 + 2^-12, -3 + 2^-11): conv0_a reads their fp16 rounding in the fp16
  mode, and seed + update adds them unrounded.  conv0_a subtracts 1000, 1 and 3 - 2^-10 from the operand, so the
  fp32 epilogue sees the bits the rounding dropped (or not)."""
  w, b = _zeros(1)
  w[0][1, 1, 1, 1, 0] = 1.0                  # relu(seed)
  w[0][1, 1, 1, 1, 1] = -1.0                 # relu(-seed)
  w[0][1, 1, 1, 1, 2] = 1.0
  b[0][2] = -1000.0                          # relu(seed - 1000)
  w[0][1, 1, 1, 1, 3] = 1.0
  b[0][3] = -1.0                             # relu(seed - 1)
  w[0][1, 1, 1, 1, 4] = -1.0
  b[0][4] = -3.0 + 2.0 ** -10                # relu(-seed - 3 + 2^-10)
  for ch in range(5):
    _pass(w, 1, ch, ch)
  w[-1][0, 0, 0, 0, 0] = -1.0
  w[-1][0, 0, 0, 1, 0] = 1.0                 # -operand(seed): seed - fp16(seed) in the fp16 mode
  w[-1][0, 0, 0, 2:5, 0] = 1.0
  seeds = np.resize(np.asarray([1000.25, 1.0 + 2.0 ** -12, -3.0 + 2.0 ** -11, 2.0], np.float32), fov)[None]
  imgs = np.zeros(fov, np.float32)[None]
  return w, b, seeds.astype(np.float32), imgs


def probe_rounding(fov):
  """conv0_a computes 2 * image + 1 = 2049, 2051, 2053, ...: odd integers above 2048 are fp16 rounding ties.  The
  identity taps of conv0_b carry the fp16 operand to conv_lom, so round-to-nearest-even, round-toward-zero and
  round-half-away give different logits."""
  w, b = _zeros(1)
  w[0][1, 1, 1, 0, 0] = 2.0
  b[0][0] = 1.0
  _pass(w, 1, 0, 0)
  w[-1][0, 0, 0, 0, 0] = 1.0
  b[-1][0] = -2048.0
  seeds = np.zeros(fov, np.float32)[None]
  imgs = (1024.0 + np.arange(int(np.prod(fov))).reshape(fov) % 8).astype(np.float32)[None]
  return w, b, seeds, imgs


def probe_subnormal(fov):
  """fp16 subnormal operands k * 2^-24: the image (k = 1 .. 7) and conv0_a's output (2k + 1) * 2^-24, fed to conv_lom
  scaled by 1.  A device that flushes fp16 subnormals gets 0 there."""
  w, b = _zeros(1)
  w[0][1, 1, 1, 0, 0] = 2.0
  b[0][0] = 2.0 ** -24
  _pass(w, 1, 0, 0)
  w[0][1, 1, 1, 0, 1] = 1.0
  _pass(w, 1, 1, 1)
  w[-1][0, 0, 0, 0, 0] = 1.0
  w[-1][0, 0, 0, 1, 0] = 1.0
  seeds = np.zeros(fov, np.float32)[None]
  imgs = ((1 + np.arange(int(np.prod(fov))).reshape(fov) % 7) * 2.0 ** -24).astype(np.float32)[None]
  return w, b, seeds, imgs


def probe_relu_order(fov):
  """ReLU at zero and below, and the order of the final sum.  conv0_b's outputs are image - 1 in {-1, 0, 1, 2}:
  conv_lom weighs them by -1/2, so a missing ReLU changes every voxel below 1.  Where the seed is 2^15, fp32 needs
  b_lom + <relu(net), w_lom> = 2^-9 + 2^-9 first: (2^15 + 2^-9) rounds back to 2^15 (a tie, to even)."""
  w, b = _zeros(1)
  _pass(w, 0, 0, 0)
  _pass(w, 0, 0, 1, 2.0 ** -9)
  _pass(w, 1, 0, 0)
  b[1][0] = -1.0
  _pass(w, 1, 1, 1)
  w[-1][0, 0, 0, 0, 0] = -0.5
  w[-1][0, 0, 0, 1, 0] = 1.0
  b[-1][0] = 2.0 ** -9
  n = int(np.prod(fov))
  imgs = (np.arange(n).reshape(fov) % 4).astype(np.float32)[None]
  seeds = np.where(np.arange(n).reshape(fov) % 3 == 0, 2.0 ** 15, 0.0).astype(np.float32)[None]
  imgs[0][seeds[0] == 2.0 ** 15] = 1.0       # image 1: net = 0, update = 2^-9 + 2^-9
  return w, b, seeds, imgs


PROBES = {'residual': probe_residual, 'bias': probe_bias, 'seed': probe_seed, 'rounding': probe_rounding,
          'subnormal': probe_subnormal, 'relu_order': probe_relu_order}

# The bugs each probe exists to catch (in the mode that can show them).
PROBE_BUGS = {'residual': [('residual_fp16', 'fp32'), ('residual_fp16', 'fp16')],
              'bias': [('bias_fp16', 'fp32'), ('bias_fp16', 'fp16')],
              'seed': [('seed_unrounded', 'fp16')],
              'rounding': [('round_toward_zero', 'fp16'), ('round_half_away', 'fp16')],
              'subnormal': [('flush_subnormal', 'fp16'), ('flush_subnormal', 'x2')],
              'relu_order': [('no_relu_before_lom', 'fp32'), ('seed_plus_bias_first', 'fp32'),
                             ('seed_plus_bias_first', 'fp16')]}


# ------------------------------------------------------------------------------------------------------------------
# The flood network
# ------------------------------------------------------------------------------------------------------------------

# Canvas image normalisation of the flood tests: u8 with mean 128 and stddev 16, so (raw - 128) / 16 is exact.
FLOOD_MEAN, FLOOD_STDDEV = 128.0, 16.0
# Flood-fill options whose float32 logits (ff.f32_logit) are small integers: init 2, pad -3, thresholds 0.
FLOOD_OPTIONS = dict(init_activation=0.8807970881462097, pad_value=0.04742586985230446,
                     move_threshold=0.5, segment_threshold=0.5)

# Reserved channels of the flood network.
E, P, N, C = 0, 1, 2, 3


def flood_net(depth, seed=1):
  """logit = relu(image) - 1 + clamp(seed, 0, 1) + sparse perturbations, exactly:

  * channel E carries relu(image) (conv0_a, identity tap) through conv0_b and the residual stream to conv_lom
    (weight 1, b_lom = -1): objects grow over voxels brighter than the mean + 1 stddev; at exactly that level the
    logit sits on the thresholds (0).
  * channels P and N carry relu(seed) and relu(-seed) to conv_lom with weights -1 and +1, which cancels the seed
    that `seed + update` adds back, and channel C = relu(seed) - relu(seed - 1) = clamp(seed, 0, 1) adds a bounded
    memory of the seed.  Every weight on a path from the seed is an integer, so a logit fed back as the next seed
    never gains fractional bits.
  * every conv also writes a few random channels from E and the other random channels (integer taps, biases multiples
    of 1/16), which conv_lom weighs by +-1/4: each layer moves some logits."""
  rng = np.random.RandomState(seed)
  w, b = _zeros(depth)
  w[0][1, 1, 1, 0, E] = 1.0
  w[0][1, 1, 1, 1, P] = 1.0
  w[0][1, 1, 1, 1, N] = -1.0
  w[0][1, 1, 1, 1, C] = 1.0
  w[0][1, 1, 1, 1, C + 1] = 1.0
  b[0][C + 1] = -1.0                         # relu(seed - 1)
  for ch in (E, P, N, C):
    _pass(w, 1, ch, ch)
  _pass(w, 1, C + 1, C, -1.0)                # net_C = relu(seed) - relu(seed - 1)
  free = list(range(8, FEAT))
  for l in range(2 * depth):
    outs = rng.choice(free, 6, replace=False)
    for co in outs:
      src = [E] + ([] if l == 0 else list(free))
      ci = int(rng.choice(src)) if l > 0 else 0
      tz, ty, tx = rng.randint(3, size=3)
      w[l][tz, ty, tx, ci, co] = np.float32(rng.choice((-1.0, 1.0)))
      b[l][co] = np.float32(rng.randint(-2, 3) / 16.0)
  wl = w[-1].reshape(FEAT)
  wl[E], wl[P], wl[N], wl[C] = 1.0, -1.0, 1.0, 1.0
  wl[rng.choice(free, 6, replace=False)] = rng.choice((-0.25, 0.25), 6)
  b[-1][0] = -1.0
  return w, b


def flood_image(cells, seed=0):
  """u8 canvas from integer cell ids (0 = membrane): membrane 96 (image -2), each cell one of 112, 144, 160, 176,
  192 (image -1, 1, 2, 3, 4).  Cells at 144 put logits exactly on the thresholds."""
  rng = np.random.RandomState(seed)
  levels = np.asarray([112, 144, 144, 160, 176, 192], np.uint8)
  lut = np.concatenate([[96], rng.choice(levels, int(cells.max()))]).astype(np.uint8)
  return lut[cells]


def flood_image_f32(vol_u8):
  return (vol_u8.astype(np.float32) - np.float32(FLOOD_MEAN)) / np.float32(FLOOD_STDDEV)
