"""A few control steps of the batched CMU corridor environment (a small target for timing and profiling runs)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dm_control_b200 import locomotion
B = int(os.environ.get('CMU_BATCH', '2048'))
env = locomotion.load('cmu_humanoid_run_walls', batch=B, seed=3)
env.physics.check_errors = False
env.reset()
g = torch.Generator(device='cuda').manual_seed(0)
a = torch.empty(B, 56, dtype=torch.float64, device='cuda')
for _ in range(int(os.environ.get('CMU_STEPS', '12'))):
  a.uniform_(-1, 1, generator=g); env.step(a)
torch.cuda.synchronize()
d = env.physics.data
print('mean ncon', float(d.ncon.double().mean()), 'mean nefc', float(d.nefc.double().mean()), 'max nefc', int(d.nefc.max()), 'warnings', d.warning.sum(0).tolist())
