"""Measures the device Atari preprocessing (SURVEY §8(f) #3): agent decisions/s for `--streams` environment streams.

  value   kernel only: raw frame pairs already resident in HBM, CUDA events around K launches
  e2e     through BatchedAtariPreprocessor.step() with HOST frames (H2D of every pooled raw frame inside the region)
  cpu     the reference's own operations on the host (np.max, np.tensordot luma, PIL bilinear resize, np.stack),
          single-threaded as the reference is, on a bounded sample

Prints one JSON line.  Roofline: HBM; algorithmic bytes per decision = 2 raw frames read + stack read + stack write."""
import argparse, ctypes as C, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--streams', type=int, default=256)
  ap.add_argument('--steps', type=int, default=200)
  ap.add_argument('--warmup', type=int, default=20)
  args = ap.parse_args()
  from dqn_zoo_b200 import _lib, parts, processors
  dev = torch.device('cuda:0')
  n, H, W = args.streams, 210, 160
  pre = processors.BatchedAtariPreprocessor(num_streams=n, device=dev, device_observations=True)
  pre._allocate((H, W, 3))
  gen = torch.Generator(device=dev).manual_seed(1)
  pre._raw.copy_(torch.randint(0, 256, pre._raw.shape, dtype=torch.uint8, device=dev, generator=gen))
  a = torch.tensor([pre._raw[e, 0].data_ptr() for e in range(n)], dtype=torch.int64, device=dev)
  b = torch.tensor([pre._raw[e, 1].data_ptr() for e in range(n)], dtype=torch.int64, device=dev)
  s = torch.tensor([pre._stacks[e].data_ptr() for e in range(n)], dtype=torch.int64, device=dev)
  counts = torch.full((n,), 4, dtype=torch.int32, device=dev)
  stream = torch.cuda.current_stream().cuda_stream

  def launch():
    nonlocal stream
    _lib.call('dz_atari_preprocess', a.data_ptr(), b.data_ptr(), n, C.byref(pre._axis_h.c), C.byref(pre._axis_v.c),
              s.data_ptr(), counts.data_ptr(), 4, C.cast(pre._luma, C.c_void_p), pre._max_band_rows, stream)

  for _ in range(args.warmup):
    launch()
  torch.cuda.synchronize()
  # the ctypes call costs more host time than the kernel runs: time a CUDA graph of `inner` launches so that the
  # device, not the Python launch rate, is what is measured
  inner = 20
  side = torch.cuda.Stream()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.stream(side):
    stream = side.cuda_stream
    launch()
    side.synchronize()
    with torch.cuda.graph(graph, stream=side):
      stream = torch.cuda.current_stream().cuda_stream
      for _ in range(inner):
        launch()
  stream = torch.cuda.current_stream().cuda_stream
  outer = max(args.steps // inner, 3)
  graph.replay()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(outer):
    graph.replay()
  e1.record()
  torch.cuda.synchronize()
  ms = e0.elapsed_time(e1) / (outer * inner)
  alg_bytes = n * (2 * H * W * 3 + 2 * 84 * 84 * 4)
  try:
    peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'MEASURED_PEAKS.json')))
    hbm = float(peaks.get('hbm_gbs', peaks.get('hbm_gbs_burst', 6650.0)))
    src = 'measured (MEASURED_PEAKS.json)'
  except Exception:
    hbm, src = 3350.0, 'H100 SXM data sheet (3.35 TB/s HBM3, 700 W)'
  # e2e: every stream emits every 4th tick; frames come from host memory
  rs = np.random.RandomState(2)
  frames = [rs.randint(0, 256, size=(H, W, 3), dtype=np.uint8) for _ in range(8)]
  pre.reset()
  ticks = 4 * max(args.steps // 20, 5)
  first = [parts.TimeStep(parts.StepType.FIRST, None, None, (frames[0], 3))] * n
  pre.step(first)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  emitted = 0
  for t in range(ticks):
    batch = [parts.TimeStep(parts.StepType.MID, 0.0, 1.0, (frames[(t + e) % 8], 3)) for e in range(n)]
    emitted += sum(o is not None for o in pre.step(batch))
  torch.cuda.synchronize()
  e2e = emitted / (time.perf_counter() - t0)
  # e2e with DEVICE-resident frames and the vectorised state machine (VectorizedAtariPreprocessor.step_arrays)
  vec = processors.VectorizedAtariPreprocessor(num_streams=n, device=dev, device_observations=True)
  dframes = torch.randint(0, 256, (n, H, W, 3), dtype=torch.uint8, device=dev, generator=gen)
  nanv = np.full(n, np.nan)
  vec.step_arrays(dframes, np.zeros(n, np.int64), nanv, nanv, np.full(n, 3))
  mid, zeros, ones, l3 = np.ones(n, np.int64), np.zeros(n), np.ones(n), np.full(n, 3)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  emitted_v = 0
  vticks = 4 * max(args.steps // 4, 20)
  for t in range(vticks):
    emitted_v += int(vec.step_arrays(dframes, mid, zeros, ones, l3)['emit'].sum())
  torch.cuda.synchronize()
  e2e_vec = emitted_v / (time.perf_counter() - t0)
  # CPU: the reference's operations (processors.py:485-500) for one stream
  from PIL import Image
  luma = [0.299, 0.587, 1 - (0.299 + 0.587)]
  stack = [np.zeros((84, 84), np.uint8)] * 4
  t0 = time.perf_counter()
  reps = 300
  for i in range(reps):
    pooled = np.max(np.stack([frames[i % 8], frames[(i + 1) % 8]], axis=0), axis=0)
    gray = np.tensordot(pooled, luma, (-1, 0)).astype(np.uint8)
    small = np.array(Image.fromarray(gray).resize((84, 84), Image.Resampling.BILINEAR), dtype=np.uint8)
    stack = stack[1:] + [small]
    obs = np.stack(stack, axis=-1)
  cpu = reps / (time.perf_counter() - t0)
  print(json.dumps({
      'metric': 'atari_preprocess_decisions_per_sec', 'value': n / (ms * 1e-3), 'unit': 'decisions/s', 'streams': n,
      'ms_per_launch': ms, 'steps': args.steps, 'warmup': args.warmup, 'dtype': 'u8 (f64 luma, int32 resample)',
      'e2e': {'value': e2e, 'unit': 'decisions/s', 'h2d_bytes_per_decision': 2 * H * W * 3,
              'note': 'BatchedAtariPreprocessor.step with host frames; host state machine + per-frame H2D included'},
      'e2e_device_frames': {'value': e2e_vec, 'unit': 'decisions/s',
                            'note': 'VectorizedAtariPreprocessor.step_arrays: frames already on the device, numpy-vectorised state '
                                    'machine, one kernel launch per tick'},
      'roofline': {'bound': 'hbm', 'achieved': alg_bytes / (ms * 1e-3) / 1e9, 'peak': hbm, 'unit': 'GB/s',
                   'frac': alg_bytes / (ms * 1e-3) / 1e9 / hbm, 'alg_bytes_per_launch': alg_bytes, 'peak_source': src, 'traffic': None},
      'cpu_baseline': {'value': cpu, 'unit': 'decisions/s', 'cores': 1, 'kind': 'reference',
                       'sample': '%d decisions of np.max + np.tensordot + PIL resize + np.stack (processors.py:485-500)' % reps}}))


if __name__ == '__main__':
  main()
