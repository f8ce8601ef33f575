"""Small profiling workload: U utterances x N frames through the C ABI (device-resident leg).
  python tools/prof_run.py U N reps lanes engine"""
import sys, os, numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uisrnn_b200 import native
from uisrnn_b200.synth import synth_utt
U = int(sys.argv[1]) if len(sys.argv) > 1 else 132
N = int(sys.argv[2]) if len(sys.argv) > 2 else 60
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 2
lanes = int(sys.argv[4]) if len(sys.argv) > 4 else 0
engine = int(sys.argv[5]) if len(sys.argv) > 5 else 0
w = dict(np.load('tests/golden/model_toy100.npz'))
m = native.NativeModel(w)
xs = np.concatenate([synth_utt(100000 + u, n_frames=N)[0] for u in range(U)]).astype(np.float32)
x = torch.from_numpy(xs).cuda()
lab = torch.empty(U * N, dtype=torch.int32, device='cuda')
off = np.arange(U + 1, dtype=np.int64) * N
for _ in range(reps):
    m.predict_device(x.data_ptr(), off, lab.data_ptr(), lanes=lanes, engine=engine)
    st = m.stats()
ph = np.array(st['phase_cycles'], dtype=np.float64)
tot = ph.sum()
print({k: v for k, v in st.items() if k != 'phase_cycles'})
print('frames/s %.0f  us/pass/cta %.1f  cols/pass %.2f' % (U * N / (st['beam_ms'] / 1e3), st['beam_ms'] * 1e3 * st['ctas'] / st['weight_passes'], st['gru_columns'] / st['weight_passes']))
print('phase share: repack %.3f gather %.3f gru %.3f w1 %.3f w2 %.3f advance %.3f land %.3f score %.3f rank %.3f assign %.3f | cycles/pass: ' % tuple(ph / tot), (ph / st['weight_passes']).round(0))
