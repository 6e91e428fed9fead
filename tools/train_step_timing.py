"""Training steps per second at the FIB-25 geometry (33^3 field of view, depth 12, batch 4), on the device and in
torch with cuDNN (bf16 autocast, fp32 master weights, the same loss and SGD update) as the baseline.

    python tools/train_step_timing.py [--out DIR] [--steps 20] [--reps 5] [--warmup 3] [--profile]

Each repeat times --steps synchronised steps with CUDA events after --warmup steps; the median and the spread over
--reps repeats are reported, with achieved TFLOP/s from `step_flops` (forward convs + dgrad of every conv but conv0_a
+ wgrad of every conv, from shapes).  --profile instead records one device step with torch.profiler and lists its
kernels (run it as a separate command).  One JSON line on stdout (and in DIR/train_step_timing[_profile].json), with
the GPU's name and power limit read in the same run.
"""

import argparse
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

FOV, DEPTH, BATCH = (33, 33, 33), 12, 4


def step_flops(fov=FOV, depth=DEPTH, batch=BATCH, features=32):
  """2 * MAC of one step: forward of every conv, dgrad of every conv but conv0_a, wgrad of every conv; conv_lom
  forward and backward."""
  v = batch * int(np.prod(fov))
  first = 27 * 2 * features
  hidden = 27 * features * features
  n_hidden = 2 * depth - 1
  fwd = first + n_hidden * hidden
  return 2 * v * (fwd + n_hidden * hidden + fwd + 3 * features)


def _gpu():
  out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=30,
                       check=True).stdout.strip().split(', ')
  return {'gpu': out[0], 'power_limit_w': float(out[1]), 'max_sm_clock_mhz': float(out[2])}


def _inputs(rng):
  shape = (BATCH,) + FOV
  return (rng.uniform(-0.5, 0.5, shape).astype(np.float32), rng.randn(*shape).astype(np.float32),
          (rng.uniform(size=shape) < 0.4).astype(np.float32))


def _time(fn, steps, reps, warmup):
  import torch
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  times = []
  for _ in range(reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
      fn()
    b.record()
    torch.cuda.synchronize()
    times.append(a.elapsed_time(b) / 1e3 / steps)
  return times


def _torch_step(w, b, seed, image, labels):
  """The same step in torch: bf16 autocast convs on cuDNN, fp32 masters, mean sigmoid cross-entropy, clipped SGD."""
  import torch
  import torch.nn.functional as F
  dev = 'cuda'
  ws = [torch.tensor(np.ascontiguousarray(x.transpose(4, 3, 0, 1, 2)), device=dev, requires_grad=True) for x in w]
  bs = [torch.tensor(x.reshape(-1), device=dev, requires_grad=True) for x in b]
  s, im, lab = (torch.tensor(x, device=dev) for x in (seed, image, labels))
  params = ws + bs
  torch.backends.cudnn.benchmark = True

  def step():
    with torch.autocast('cuda', dtype=torch.bfloat16):
      net = torch.stack([im, s], 1)
      net = F.conv3d(F.relu(F.conv3d(net, ws[0], bs[0], padding=1)), ws[1], bs[1], padding=1)
      for m in range(1, DEPTH):
        net = F.conv3d(F.relu(F.conv3d(F.relu(net), ws[2 * m], bs[2 * m], padding=1)), ws[2 * m + 1],
                       bs[2 * m + 1], padding=1) + net
    net = F.relu(net.float())
    logits = s + F.conv3d(net, ws[-1], bs[-1])[:, 0]
    loss = F.binary_cross_entropy_with_logits(logits, lab)
    grads = torch.autograd.grad(loss, params)
    with torch.no_grad():
      for p, g in zip(params, grads):
        p.sub_(0.001 * g.clamp(-0.7, 0.7))
  return step


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--reps', type=int, default=5)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--profile', action='store_true')
  args = ap.parse_args()
  import torch
  from ffn_b200 import tf_checkpoint
  from ffn_b200.training.trainer import Trainer
  if not torch.cuda.is_available():
    raise SystemExit('no CUDA device: nothing to time')
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(REPO, 'tests', 'golden', 'fib25_convstack.npz'))
  seed, image, labels = _inputs(np.random.RandomState(0))
  tr = Trainer(w, b, FOV, batch_size=BATCH)
  dev_step = lambda: tr.step(seed, image, labels)
  res = dict(_gpu(), fov=FOV, depth=DEPTH, batch=BATCH, flop_per_step=step_flops())
  if args.profile:
    from torch.profiler import ProfilerActivity, profile
    for _ in range(args.warmup):
      dev_step()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      dev_step()
      torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
      if e.device_type.name == 'CUDA':
        kern[e.name] = kern.get(e.name, 0.0) + e.device_time / 1e3
    res['kernel_ms'] = dict(sorted(kern.items(), key=lambda kv: -kv[1]))
  else:
    for name, fn in (('device', dev_step), ('torch_cudnn_bf16', _torch_step(w, b, seed, image, labels))):
      t = _time(fn, args.steps, args.reps, args.warmup)
      med = float(np.median(t))
      res[name] = {'steps_per_s': 1.0 / med, 'ms_median': med * 1e3, 'ms_min': min(t) * 1e3, 'ms_max': max(t) * 1e3,
                   'tflops': step_flops() / med / 1e12}
  tr.close()
  line = json.dumps(res)
  print(line)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'train_step_timing%s.json' % ('_profile' if args.profile else '')), 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
