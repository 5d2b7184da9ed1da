"""Per-kernel CUDA-event times of the 1 x 1101 heads and of a single-scan leg (development aid for
parameter sweeps: OVN_* environment switches are read once per process).  The leg is timed twice: warm
(legs back to back, its weights and activations stay in L2) and cold (a heads_1vsN call between two legs,
as in the query step, which streams over 1 GB and evicts L2)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from overlapnet_b200.engine import Engine
from oracle import network as N

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
n = 1101
eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=n)
eng.load_weights(N.glorot_weights(4, MODEL, seed=0))
g = torch.Generator(device='cuda').manual_seed(0)
bank = torch.rand((n, 360, 128), device='cuda', generator=g)
eng.bank_prepare(bank, 0, n)
for _ in range(3): eng.heads_1vsN(bank, bank[0], n_cand=n)
torch.cuda.synchronize()
eng.profile_enable(True)
for _ in range(10): eng.heads_1vsN(bank, bank[0], n_cand=n)
torch.cuda.synchronize()
out = []
for k in ('delta_conv1', 'conv2', 'conv3', 'corr'):
  ms, c = eng.profile_read(k)
  out.append('%s %.4f' % (k, ms / max(c, 1)))
x = torch.rand((1, 64, 900, 4), device='cuda', generator=g) * 30
for _ in range(3): eng.leg(x)
torch.cuda.synchronize()
eng.profile_read('leg')
for _ in range(20): eng.leg(x)
torch.cuda.synchronize()
ms, c = eng.profile_read('leg')
out.append('leg_warm %.4f' % (ms / max(c, 1)))
for _ in range(10):
  eng.heads_1vsN(bank, bank[0], n_cand=n)
  eng.leg(x)
torch.cuda.synchronize()
ms, c = eng.profile_read('leg')
out.append('leg_cold %.4f' % (ms / max(c, 1)))
print(os.environ.get('TAG', ''), torch.cuda.get_device_name(), ' '.join(out))
