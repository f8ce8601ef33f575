"""A/B of the beam-kernel engines on bench.py's workload (device-resident): frames/s, kernel ms, phase shares.
  python tools/tc_bench.py [U ...]      e.g.  python tools/tc_bench.py 264 792"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ['repack(P4)', 'gather', 'GRU', 'W1', 'W2', 'advance', 'landing(P0)', 'score(P1)', 'rank(P2)', 'assign(P3)']


def main():
  import torch
  from uisrnn_b200 import native
  from uisrnn_b200.synth import synth_utt
  native.load_library()
  model = native.NativeModel(dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'model_toy100.npz'))))
  sizes = [int(a) for a in sys.argv[1:]] or [264, 792]
  n_frames = int(os.environ.get('TC_BENCH_FRAMES', '500'))
  umax = max(sizes)
  xs = np.concatenate([synth_utt(100000 + u, n_frames=n_frames)[0] for u in range(umax)]).astype(np.float32)
  x_dev = torch.from_numpy(xs).cuda()
  ref = {}
  for U in sizes:
    off = np.arange(U + 1, dtype=np.int64) * n_frames
    lab = torch.empty(U * n_frames, dtype=torch.int32, device='cuda')
    for engine in [int(v) for v in os.environ.get('TC_BENCH_ENGINES', '1,2').split(',')]:
      for lanes in ([0] if engine == 1 else [int(v) for v in os.environ.get('TC_BENCH_LANES', '0,4,6').split(',')]):
        try:
          for _ in range(2):
            model.predict_device(x_dev.data_ptr(), off, lab.data_ptr(), engine=engine, lanes=lanes)
            st = model.stats()
        except native.NativeError as err:
          print(json.dumps({'U': U, 'engine': engine, 'lanes': lanes, 'error': str(err)[:200]}), flush=True)
          continue
        got = lab.cpu().numpy().copy()
        if engine == 1:
          ref[U] = got
        tot = float(sum(st['phase_cycles'])) or 1.0
        print(json.dumps({
            'U': U, 'engine': st['engine'], 'lanes': st['lanes'], 'tc_columns': st['tc_columns'], 'ctas': st['ctas'],
            'beam_ms': round(st['beam_ms'], 3), 'prepass_ms': round(st['prepass_ms'], 3),
            'frames_per_s': round(U * n_frames / ((st['beam_ms'] + st['prepass_ms']) / 1e3)),
            'us_per_lane_step': round(1e3 * st['beam_ms'] * st['ctas'] * st['lanes'] / max(1, st['beam_steps']), 2),
            'cols_per_pass': round(st['gru_columns'] / max(1, st['weight_passes']), 2),
            'passes': st['weight_passes'], 'labels_equal_ffma': bool(np.array_equal(got, ref.get(U, got))),
            'mismatching_frames': int((got != ref.get(U, got)).sum()),
            'phase_share': {n: round(c / tot, 3) for n, c in zip(PHASES, st['phase_cycles'])},
            'phase_us_per_cta_step': {n: round(c / 1980.0 / max(1, st['beam_steps'] / max(1, st['lanes'])), 2)
                                      for n, c in zip(PHASES, st['phase_cycles'])},
            'tc_pass_us_per_pass': {n: round(c / 1980.0 / max(1, st['weight_passes']), 2) for n, c in
                                    zip(['wait_tma', 'wait_mma', 'stage_b_operand', 'pass'], st['tc_cycles'])}}),
              flush=True)


if __name__ == '__main__':
  main()
