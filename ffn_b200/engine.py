"""Python handles over the C ABI: `Engine` (device + packed model) and `DeviceCanvas`
(HBM-resident flood-fill state).  The reference-facing classes in ``ffn_b200.inference`` sit on
top of these; nothing here computes on the CPU.
"""

from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
from scipy.special import logit

from . import _lib


def f32_logit(p: float) -> float:
  """float32 proto field after Canvas.__init__ stored logit(p) back (inference.py:186-195)."""
  return float(np.float32(logit(float(np.float32(p)))))


def make_options(init_activation=0.95, pad_value=0.05, move_threshold=0.9, segment_threshold=0.6,
                 disco_seed_threshold=0.0, min_boundary_dist_zyx=(1, 1, 1), min_segment_size=1000,
                 policy_score_threshold: Optional[float] = None) -> _lib.Options:
  """Builds FfnOptions from probability-space InferenceOptions values."""
  o = _lib.Options()
  o.init_activation = f32_logit(init_activation)
  o.pad_value = f32_logit(pad_value)
  o.move_threshold = f32_logit(move_threshold)
  o.segment_threshold = f32_logit(segment_threshold)
  o.disco_seed_threshold = float(np.float32(disco_seed_threshold))
  if policy_score_threshold is None:  # movement.get_policy_fn (movement.py:241-242)
    policy_score_threshold = float(logit(float(np.float32(move_threshold))))
  o.policy_score_threshold = float(policy_score_threshold)
  o.min_boundary_dist_zyx = _lib.i3(min_boundary_dist_zyx)
  o.min_segment_size = int(min_segment_size)
  return o


class Engine:
  """One per GPU: owns the packed ConvStack3DFFNModel weights and the step workspace."""

  def __init__(self, weights_dhwio: Sequence[np.ndarray], biases: Sequence[np.ndarray],
               fov_zyx=(33, 33, 33), deltas_zyx=(8, 8, 8), device: int = 0,
               compute_mode: int = _lib.COMPUTE_FP16_TC, num_ctas: int = 0):
    self._lib = _lib.load()
    depth = (len(weights_dhwio) - 1) // 2
    if len(weights_dhwio) != 2 * depth + 1 or len(biases) != len(weights_dhwio):
      raise ValueError('expected 2*depth+1 weight/bias arrays')
    self.depth = depth
    self.fov_zyx = tuple(int(v) for v in fov_zyx)
    self.deltas_zyx = tuple(int(v) for v in deltas_zyx)
    self.device = int(device)
    ws = [np.ascontiguousarray(w, dtype=np.float32) for w in weights_dhwio]
    bs = [np.ascontiguousarray(b, dtype=np.float32) for b in biases]
    for i, w in enumerate(ws[:-1]):
      want = (3, 3, 3, 2 if i == 0 else 32, 32)
      if w.shape != want:
        raise ValueError('layer %d weights have shape %r, expected %r' % (i, w.shape, want))
    if ws[-1].size != 32:
      raise ValueError('conv_lom weights must have 32 inputs and 1 output')
    desc = _lib.ModelDesc()
    desc.fov_zyx = _lib.i3(self.fov_zyx)
    desc.deltas_zyx = _lib.i3(self.deltas_zyx)
    desc.depth = depth
    desc.features = 32
    wp = (C.c_void_p * len(ws))(*[w.ctypes.data for w in ws])
    bp = (C.c_void_p * len(bs))(*[b.ctypes.data for b in bs])
    h = C.c_void_p()
    _lib.check(self._lib.ffn_engine_create(self.device, C.byref(desc), wp, bp, int(compute_mode),
                                            C.byref(h)))
    self._h = h
    self.compute_mode = int(compute_mode)
    if num_ctas:
      self.set_grid(num_ctas)

  def close(self):
    if getattr(self, '_h', None):
      self._lib.ffn_engine_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  def set_grid(self, num_ctas: int):
    """SM budget of this engine's persistent kernel (0 = whole GPU); see ffn_engine_set_grid."""
    _lib.check(self._lib.ffn_engine_set_grid(self._h, int(num_ctas)))

  def set_chains(self, max_chains: int):
    """Objects / patches in flight at once in the persistent kernel (1..4, 0 = default 4); see ffn_engine_set_chains."""
    _lib.check(self._lib.ffn_engine_set_chains(self._h, int(max_chains)))

  def set_compute_mode(self, mode: int):
    _lib.check(self._lib.ffn_engine_set_compute_mode(self._h, int(mode)))
    self.compute_mode = int(mode)

  def info(self) -> dict:
    buf = (C.c_int64 * 8)()
    _lib.check(self._lib.ffn_engine_info(self._h, buf))
    keys = ('sm_count', 'grid', 'smem_bytes', 'tiles', 'rows', 'fov_voxels', 'launches', 'last_kernel_ns')
    return dict(zip(keys, [int(v) for v in buf]))

  PROFILE_SLOTS = ('barrier_wait', 'act_tma_wait', 'weight_wait', 'mma', 'unused4', 'epi_body',
                   'stage', 'paste', 'leader', 'steps', 'kernel', 'conv_layers', 'leader_policy', 'leader_pops',
                   'chain_barrier_wait', 'unused')

  def enable_profiling(self, on: bool = True):
    _lib.check(self._lib.ffn_engine_profile(self._h, None, 1 if on else 0))

  def profile(self, reset: bool = True) -> dict:
    """Device cycle counters of CTA 0 and of the last CTA (see ffn_engine_profile)."""
    buf = (C.c_int64 * 32)()
    _lib.check(self._lib.ffn_engine_profile(self._h, buf, 1 if reset else 0))
    return {'cta0': dict(zip(self.PROFILE_SLOTS, [int(v) for v in buf[:16]])),
            'cta_last': dict(zip(self.PROFILE_SLOTS, [int(v) for v in buf[16:32]]))}

  def trace(self, reset: bool = True) -> np.ndarray:
    """[8 events][2048 tiles] SM-clock timeline of CTA 1 (see ffn_engine_trace); needs enable_profiling()."""
    buf = np.zeros((8, 2048), dtype=np.int64)
    _lib.check(self._lib.ffn_engine_trace(self._h, buf.ctypes.data_as(C.POINTER(C.c_int64)), buf.size, 1 if reset else 0))
    return buf

  def predict(self, seed: np.ndarray, image: np.ndarray) -> np.ndarray:
    """(Z,Y,X) or (B,Z,Y,X) float32 patches -> logits of the same shape (executor.py:134-139)."""
    seed = np.ascontiguousarray(seed, dtype=np.float32)
    image = np.ascontiguousarray(image, dtype=np.float32)
    if seed.shape != image.shape:
      raise ValueError('seed and image shapes differ')
    single = seed.ndim == 3
    if seed.shape[-3:] != self.fov_zyx:
      raise ValueError('patch shape %r does not match the model FoV %r' % (seed.shape[-3:], self.fov_zyx))
    batch = 1 if single else seed.shape[0]
    out = np.empty_like(seed)
    _lib.check(self._lib.ffn_predict(self._h, _lib.ptr(seed), _lib.ptr(image), batch, _lib.ptr(out)))
    return out


class DeviceCanvas:
  """HBM-resident seed / segmentation / probability canvases plus the movement-policy state."""

  def __init__(self, engine: Engine, image: np.ndarray, options: _lib.Options,
               image_mean: float = 0.0, image_stddev: float = 1.0,
               keep_probability_maps: bool = True):
    self.engine = engine
    self._lib = engine._lib
    if image.ndim != 3:
      raise ValueError('image must be (z, y, x)')
    if image.dtype == np.uint8:
      dtype = _lib.IMAGE_U8
      img = np.ascontiguousarray(image)
    else:
      dtype = _lib.IMAGE_F32
      img = np.ascontiguousarray(image, dtype=np.float32)
    self.shape = tuple(int(s) for s in img.shape)
    self.options = options
    h = C.c_void_p()
    _lib.check(self._lib.ffn_canvas_create(engine._h, _lib.ptr(img), dtype, _lib.i3(self.shape),
                                            float(image_mean), float(image_stddev), C.byref(options),
                                            1 if keep_probability_maps else 0, C.byref(h)))
    self._h = h
    self.keep_probability_maps = keep_probability_maps

  def close(self):
    if getattr(self, '_h', None):
      self._lib.ffn_canvas_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  # -- masks ---------------------------------------------------------------------------------
  def set_mask(self, which: int, mask: Optional[np.ndarray]):
    if mask is None:
      _lib.check(self._lib.ffn_canvas_set_mask(self._h, which, None))
      return
    m = np.ascontiguousarray(np.asarray(mask) != 0, dtype=np.uint8)
    if m.shape != self.shape:
      raise ValueError('mask shape mismatch')
    _lib.check(self._lib.ffn_canvas_set_mask(self._h, which, _lib.ptr(m)))

  # -- hot loop ------------------------------------------------------------------------------
  def segment_at(self, start_zyx, reset: bool = True, max_steps: int = 0, keep_seed: bool = False) -> _lib.SegStats:
    """reset=False resumes the object in flight; keep_seed=True starts a new object WITHOUT init_seed / extent
    reset (Canvas.reset_seed_per_segment == False, inference.py:486-490)."""
    st = _lib.SegStats()
    _lib.check(self._lib.ffn_canvas_segment_at(self._h, _lib.i3(start_zyx), (2 if keep_seed else 1) if reset else 0,
                                                int(max_steps), C.byref(st)))
    return st

  def segment_all(self, seeds_zyx: np.ndarray, origins_cap: Optional[int] = None,
                  overlaps_cap: Optional[int] = None):
    seeds = np.ascontiguousarray(np.asarray(seeds_zyx).reshape(-1, 3), dtype=np.int32)
    n = seeds.shape[0]
    origins_cap = int(origins_cap or max(n, 1))
    overlaps_cap = int(overlaps_cap or max(8 * n, 1024))
    origins = (_lib.Origin * origins_cap)()
    overlaps = (_lib.Overlap * overlaps_cap)()
    n_o, n_v = C.c_int64(0), C.c_int64(0)
    ctr = _lib.Counters()
    _lib.check(self._lib.ffn_canvas_segment_all(
        self._h, _lib.ptr(seeds), n, C.cast(origins, C.c_void_p), origins_cap, C.byref(n_o),
        C.cast(overlaps, C.c_void_p), overlaps_cap, C.byref(n_v), C.byref(ctr)))
    if n_o.value > origins_cap or n_v.value > overlaps_cap:
      raise RuntimeError('origins/overlaps output capacity exceeded (%d/%d, %d/%d)' %
                         (n_o.value, origins_cap, n_v.value, overlaps_cap))
    return list(origins[:n_o.value]), list(overlaps[:n_v.value]), ctr

  def update_at(self, pos_zyx) -> np.ndarray:
    out = np.empty(self.engine.fov_zyx, dtype=np.float32)
    _lib.check(self._lib.ffn_canvas_update_at(self._h, _lib.i3(pos_zyx), _lib.ptr(out)))
    return out

  def init_seed(self, pos_zyx):
    _lib.check(self._lib.ffn_canvas_init_seed(self._h, _lib.i3(pos_zyx)))

  # -- state I/O -----------------------------------------------------------------------------
  _DTYPES = {_lib.ARRAY_SEED: np.float32, _lib.ARRAY_SEGMENTATION: np.int32,
             _lib.ARRAY_QPROB: np.uint8, _lib.ARRAY_IMAGE: np.float32}

  def read(self, which: int, lo=None, size=None) -> np.ndarray:
    lo = (0, 0, 0) if lo is None else tuple(int(v) for v in lo)
    size = tuple(s - l for s, l in zip(self.shape, lo)) if size is None else tuple(int(v) for v in size)
    out = np.empty(size, dtype=self._DTYPES[which])
    _lib.check(self._lib.ffn_canvas_read(self._h, which, _lib.i3(lo), _lib.i3(size), _lib.ptr(out)))
    return out

  def write(self, which: int, data: np.ndarray, lo=(0, 0, 0)):
    arr = np.ascontiguousarray(data, dtype=self._DTYPES[which])
    _lib.check(self._lib.ffn_canvas_write(self._h, which, _lib.i3(lo), _lib.i3(arr.shape), _lib.ptr(arr)))

  def counters(self) -> _lib.Counters:
    c = _lib.Counters()
    _lib.check(self._lib.ffn_canvas_get_counters(self._h, C.byref(c)))
    return c

  def spec_stats(self) -> dict:
    """Early-run bookkeeping of the last segment_all (see ffn_canvas_spec_stats)."""
    buf = (C.c_int64 * 8)()
    _lib.check(self._lib.ffn_canvas_spec_stats(self._h, buf))
    return dict(zip(('early_runs', 'early_runs_discarded', 'steps_discarded', 'steps_executed', 'rounds',
                     'chain_rounds_free', 'chain_rounds_waiting', 'chains'), [int(v) for v in buf]))

  def set_resume(self, iters: int, min_pos, max_pos):
    _lib.check(self._lib.ffn_canvas_set_resume(self._h, int(iters), _lib.i3(min_pos), _lib.i3(max_pos)))

  def start_trace(self, capacity: int = 1 << 20):
    self._trace_cap = int(capacity)
    _lib.check(self._lib.ffn_canvas_trace(self._h, int(capacity), None, None))

  def get_trace(self, with_total: bool = False):
    """[n, 4] int32 rows (type, z, y, x); see ffn_canvas_trace.  `with_total` also returns the number of
    events produced (more than n when the log overflowed)."""
    buf = np.empty((getattr(self, '_trace_cap', 0), 4), dtype=np.int32)   # only the produced rows are filled
    n = C.c_int64(0)
    _lib.check(self._lib.ffn_canvas_trace(self._h, 0, _lib.ptr(buf), C.byref(n)))
    events = buf[:min(int(n.value), buf.shape[0])]
    return (events, int(n.value)) if with_total else events

  def seed_peaks(self, voxel_size_zyx=(1, 1, 1), noise: Optional[np.ndarray] = None, cap: Optional[int] = None):
    """Device PolicyPeaks: returns the peak coordinates [N, 3] (z, y, x), lexicographically sorted."""
    cap = int(cap or max(self.shape[0] * self.shape[1] * self.shape[2] // 64, 4096))
    vs = (C.c_float * 3)(*[float(v) for v in voxel_size_zyx])
    while True:
      out = np.empty((cap, 3), dtype=np.int32)
      n = C.c_int64(0)
      nz = None
      if noise is not None:
        nz = np.ascontiguousarray(noise, dtype=np.float64)
        if nz.shape != self.shape:
          raise ValueError('noise shape mismatch')
      _lib.check(self._lib.ffn_canvas_seed_peaks(self._h, vs, _lib.ptr(nz) if nz is not None else None, _lib.ptr(out),
                                                  cap, C.byref(n)))
      if n.value <= cap:
        break
      cap = int(n.value)
    coords = out[:n.value]
    order = np.lexsort((coords[:, 2], coords[:, 1], coords[:, 0]))
    return coords[order]

  def set_max_id(self, max_id: int):
    _lib.check(self._lib.ffn_canvas_set_max_id(self._h, int(max_id)))

  def policy_state(self):
    """Returns (queue [(score, z, y, x)], done-set [(qz, qy, qx)], start) — movement.py:180-184."""
    ql, dl = C.c_int64(0), C.c_int64(0)
    _lib.check(self._lib.ffn_canvas_policy_state_size(self._h, C.byref(ql), C.byref(dl)))
    queue = np.zeros((ql.value, 4), dtype=np.float64)
    done = np.zeros((dl.value, 3), dtype=np.int32)
    start = (C.c_int32 * 3)()
    _lib.check(self._lib.ffn_canvas_policy_state_get(self._h, _lib.ptr(queue), _lib.ptr(done), start))
    return queue, done, tuple(int(v) for v in start)

  def set_policy_state(self, queue: np.ndarray, done: np.ndarray, start_zyx):
    queue = np.ascontiguousarray(np.asarray(queue, dtype=np.float64).reshape(-1, 4))
    done = np.ascontiguousarray(np.asarray(done, dtype=np.int32).reshape(-1, 3))
    _lib.check(self._lib.ffn_canvas_policy_state_set(self._h, _lib.ptr(queue), queue.shape[0],
                                                      _lib.ptr(done), done.shape[0], _lib.i3(start_zyx)))

  def device_ptr(self, which: int):
    p, n = C.c_void_p(), C.c_int64(0)
    _lib.check(self._lib.ffn_canvas_device_ptr(self._h, which, C.byref(p), C.byref(n)))
    return int(p.value), int(n.value)

  def add_id_offset(self, offset: int):
    _lib.check(self._lib.ffn_canvas_add_id_offset(self._h, int(offset)))


def selftest(variant: int, device: int = 0, n_out: int = 8) -> list:
  lib = _lib.load()
  out = (C.c_double * n_out)()
  _lib.check(lib.ffn_selftest_umma(int(device), int(variant), out, n_out))
  return [float(v) for v in out]
