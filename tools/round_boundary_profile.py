"""The round boundary of Canvas.segment_all on the bench canvas (profiled kernel build), split by phase: what the
leader (CTA 0) spends between the grid barrier and the release of the round flag, and what the last CTA spends
pasting and waiting for that flag.  Needs a GPU.   python tools/round_boundary_profile.py [n=250] [chains...]

One JSON line per chain count: cycles per round of every boundary counter on CTA 0 and on the last CTA, the
scheduler's round statistics, executed FoV steps per round, and the card the cycles were counted on (name, power
limit, median SM clock while the unprofiled run was going)."""
import json, os, sys
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import numpy as np
import bench
from ffn_b200 import engine as eng, tf_checkpoint

BOUNDARY = ('barrier_wait', 'leader', 'leader_copy_in', 'leader_policy', 'leader_pops', 'leader_advance',
            'leader_copy_out', 'paste', 'round_flag_wait', 'stage', 'face_reduce', 'conv_layers', 'kernel')

W, B = tf_checkpoint.load_convstack_npz(os.path.join(REPO, 'tests', 'golden', 'fib25_convstack.npz'))
n = int(sys.argv[1]) if len(sys.argv) > 1 else 250
chain_list = [int(a) for a in sys.argv[2:]] or [1, 4]
e = eng.Engine(W, B, (33, 33, 33), (8, 8, 8))   # raises without a GPU
vol = bench.make_volume((n, n, n), 0)
cv = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
coords = cv.seed_peaks((1, 1, 1), np.random.RandomState(seed=42).rand(*cv.shape))
cv.close()
m = np.asarray((16, 16, 16))[None]
seeds = np.ascontiguousarray(coords[np.all((coords - m >= 0) & (coords + m < n), axis=1)], dtype=np.int32)
for chains in chain_list:
  e.set_chains(chains)
  for prof in (False, True):
    e.enable_profiling(prof)
    if prof:
      e.profile(reset=True)
    cv = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
    sampler = bench.ClockSampler(0)
    if not prof:
      sampler.start()
      sampler.wait_ready()
    _, _, ctr = cv.segment_all(seeds, overlaps_cap=1 << 18)
    sp = cv.spec_stats()
    cv.close()
    if not prof:
      clocks = sampler.stop()
      plain = float(ctr.device_seconds)
      continue
    p = e.profile()
    rounds = max(sp['rounds'], 1)
    out = {'chains': chains, 'gpu': clocks.get('gpu'), 'power_limit_w': clocks.get('power_limit_w'),
           'sm_mhz': clocks.get('sm_mhz'), 'plain_dev_s': round(plain, 4),
           'profiled_dev_s': round(float(ctr.device_seconds), 4), 'us_per_round': round(1e6 * plain / rounds, 2),
           'rounds': rounds, 'steps_executed': sp['steps_executed'],
           'chain_rounds_free': sp['chain_rounds_free'], 'chain_rounds_waiting': sp['chain_rounds_waiting'],
           'steps_per_round': round(sp['steps_executed'] / rounds, 3),
           'cta0_cycles_per_round': {k: round(p['cta0'][k] / rounds) for k in BOUNDARY},
           'cta_last_cycles_per_round': {k: round(p['cta_last'][k] / rounds) for k in BOUNDARY}}
    print(json.dumps(out), flush=True)
e.close()
