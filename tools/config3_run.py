"""BASELINE config 3 (beam_size=30, look_ahead=2, hidden=512) throughput probe, device-resident."""
import sys, os, numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uisrnn_b200 import native
from uisrnn_b200.synth import synth_utt
U = int(sys.argv[1]) if len(sys.argv) > 1 else 132
N = int(sys.argv[2]) if len(sys.argv) > 2 else 100
beam = int(sys.argv[3]) if len(sys.argv) > 3 else 30
la = int(sys.argv[4]) if len(sys.argv) > 4 else 2
w = dict(np.load('tests/golden/model_toy100.npz'))
m = native.NativeModel(w)
xs = np.concatenate([synth_utt(1000 + u, n_frames=N)[0] for u in range(U)]).astype(np.float32)
x = torch.from_numpy(xs).cuda()
lab = torch.empty(U * N, dtype=torch.int32, device='cuda')
off = np.arange(U + 1, dtype=np.int64) * N
for _ in range(2):
    m.predict_device(x.data_ptr(), off, lab.data_ptr(), beam_size=beam, look_ahead=la)
    st = m.stats()
print({k: v for k, v in st.items() if k != 'phase_cycles'})
print('config3-like: U=%d N=%d beam=%d look_ahead=%d: %.0f frames/s, %.2f ms, cols/step %.1f, passes/step %.2f' % (
    U, N, beam, la, U * N / (st['beam_ms'] / 1e3), st['beam_ms'], st['gru_columns'] / st['beam_steps'], st['weight_passes'] / st['beam_steps']))
