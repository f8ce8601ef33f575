"""Few-utterance (latency) regime: frames/s for U = 1, 8, 32, 64 with the cluster mode off / auto / forced."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from uisrnn_b200 import native
from uisrnn_b200.synth import synth_utt
N = 500
m = native.NativeModel(dict(np.load('tests/golden/model_toy100.npz')))
for U in (1, 2, 4, 8, 32, 64):
  xs = torch.from_numpy(np.concatenate([synth_utt(1000 + u, n_frames=N)[0] for u in range(U)]).astype(np.float32)).cuda()
  lab = torch.empty(U * N, dtype=torch.int32, device='cuda')
  off = np.arange(U + 1, dtype=np.int64) * N
  ref = None
  for cluster in (-1, 0, 2, 4, 8, 32):
    if cluster > 0 and cluster < 32 and U * cluster > 132:
      continue
    if cluster == 32 and U > 8:
      continue
    for _ in range(2):
      m.predict_device(xs.data_ptr(), off, lab.data_ptr(), cluster=cluster)
      st = m.stats()
    got = lab.cpu().numpy().copy()
    if ref is None:
      ref = got
    print('U=%-3d cluster opt %2d -> used %d ctas %3d: %8.0f frames/s (%.2f ms)  labels %s' % (
        U, cluster, st['cluster'], st['ctas'], U * N / ((st['beam_ms'] + st['prepass_ms']) / 1e3),
        st['beam_ms'] + st['prepass_ms'], 'same' if np.array_equal(ref, got) else 'DIFFER'), flush=True)
