"""Per-kernel device time of the bench workload (suite.humanoid:run, B = 8192) under torch.profiler.

Start states as bench.py: the task's initialize_episode + 21 settle env-steps with uniform(-1, 1) actions; then
`--steps` eager control steps (no CUDA graph, so every kernel is its own profiler event) are traced. Prints one JSON
line: the card, per kernel name (template arguments included) its device time per control step, share of the kernel
total and launches per control step, the acceleration kernels' time per row bucket, and the contact load of the traced
steps (bucket populations, mean nefc, mean solver iterations). Run it on its own: tracing slows the host, so its times are not the benchmark's.

  python tools/acc_profile.py [--batch 8192] [--steps 10] [--out DIR]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(',')]
    return dict(name=name, power_limit=power, max_sm_clock=clock)
  except Exception as ex:            # the numbers below still stand; the card is then unnamed
    return dict(error=repr(ex))


def per_bucket_launches(trace, steps):
  """Acceleration-kernel time per row bucket. Every (environment group, bucket) pair launches on a stream of its own,
  in the order group 0: buckets 0, 1, ..; group 1: buckets 0, 1, .. (b200mj_step), so the streams ranked by their first
  launch give the buckets; bucket 0 shares its stream with its group's position kernel."""
  ev = json.load(open(trace))['traceEvents']
  streams, pos_streams = {}, set()
  for e in ev:
    if e.get('cat') != 'kernel':
      continue
    a = e.get('args', {})
    if 'pos_kernel' in e.get('name', ''):
      pos_streams.add(a.get('stream'))
    if 'acc_kernel' in e.get('name', ''):
      s = streams.setdefault(a.get('stream'), dict(us=0.0, n=0, first=float('inf'), stream=a.get('stream')))
      s['us'] += e.get('dur', 0.0); s['n'] += 1; s['first'] = min(s['first'], a.get('correlation', e.get('ts', 0)))
  ranked = sorted(streams.values(), key=lambda s: s['first'])
  nb = max(1, len(ranked) // 2)
  out = []
  for b in range(nb):
    group = [s for i, s in enumerate(ranked) if i % nb == b]
    out.append(dict(bucket=b, ms_per_control_step=round(sum(s['us'] for s in group) / steps / 1e3, 4),
                    launches_per_control_step=sum(s['n'] for s in group) / steps,
                    on_position_stream=all(s['stream'] in pos_streams for s in group)))
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=8192)
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--settle', type=int, default=21)
  ap.add_argument('--out', help='directory for the chrome trace (optional)')
  args = ap.parse_args()

  import torch
  from torch.profiler import ProfilerActivity, profile
  from dm_control_b200 import suite

  dev = torch.device('cuda', 0)
  env = suite.load('humanoid', 'run', batch=args.batch, seed=1000, device=dev)
  env.physics.check_errors = False
  env._graph_task_ops = False
  env._graph_step = False
  env.reset()
  phys = env.physics
  gen = torch.Generator(device=dev).manual_seed(1234)
  act = torch.empty(args.batch, phys.model.nu, dtype=torch.float64, device=dev)
  for _ in range(args.settle):
    act.uniform_(-1, 1, generator=gen); env.step(act)
  torch.cuda.synchronize()

  snaps = []
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.steps):
      act.uniform_(-1, 1, generator=gen); env.step(act)
      snaps.append(tuple(getattr(phys.data, f).clone().double() for f in ('ncon', 'nefc', 'solver_niter')))
    torch.cuda.synchronize()
  out_dir = args.out or tempfile.mkdtemp(prefix='acc_profile_')
  os.makedirs(out_dir, exist_ok=True)
  trace = os.path.join(out_dir, 'acc_profile.pt.trace.json')
  prof.export_chrome_trace(trace)
  launches = per_bucket_launches(trace, args.steps)
  if not args.out:
    shutil.rmtree(out_dir, ignore_errors=True)

  kernels = {}
  for ev in prof.events():
    if ev.device_type != torch.autograd.DeviceType.CUDA or ev.name.startswith(('Memcpy', 'Memset')):
      continue
    k = kernels.setdefault(ev.name, [0.0, 0])
    k[0] += ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
    k[1] += 1
  total = sum(v[0] for v in kernels.values())
  rows = sorted(((n, v[0] / args.steps / 1e3, v[0] / total, v[1] / args.steps) for n, v in kernels.items()), key=lambda r: -r[1])

  ncon = torch.cat([s[0] for s in snaps]); nefc = torch.cat([s[1] for s in snaps]); niter = torch.cat([s[2] for s in snaps])
  caps = [b['rows'] for b in phys.describe().get('acc_buckets', [])]
  pops, lo = [], -1
  for c in caps:
    pops.append(float(((nefc > lo) & (nefc <= c)).double().mean())); lo = c
  out = dict(card=card(), batch=args.batch, control_steps=args.steps, n_sub_steps=env.n_sub_steps,
             kernel_ms_per_control_step=total / args.steps / 1e3,
             kernels=[dict(name=n, ms_per_control_step=round(ms, 4), share=round(s, 4), launches_per_control_step=l)
                      for n, ms, s, l in rows],
             acc_buckets=[dict(b, rows=caps[b['bucket']] if b['bucket'] < len(caps) else None) for b in launches],
             contact_load=dict(mean_ncon=float(ncon.mean()), mean_nefc=float(nefc.mean()), mean_niter=float(niter.mean()),
                               bucket_caps=caps, bucket_populations=pops))
  print(json.dumps(out))


if __name__ == '__main__':
  main()
