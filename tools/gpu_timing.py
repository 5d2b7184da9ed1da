"""What every timing tool needs, written once: the card a number was measured on, CUDA-event step timers and
spawned data-parallel ranks.  A speed claim in this project comes with the card's name and power limit read in the
same run (DESIGN.md section 5), so every tool reads them through card()."""
import json
import os
import socket
import subprocess
import tempfile
import uuid

import numpy as np
import torch


def require_cuda(tool):
  """Exit with a message when there is no CUDA device: a time taken on the CPU says nothing about the GPU."""
  if not torch.cuda.is_available():
    raise SystemExit('%s needs a CUDA device' % tool)


def nvidia_smi(fields, device=None):
  """nvidia-smi's ``--query-gpu`` values of ``fields`` for CUDA device ``device`` (default: the current one).  The
  card is named by its UUID, so the values are those of the device in use whatever CUDA_VISIBLE_DEVICES says.  When
  nvidia-smi fails every value is 'unknown (<reason>)'."""
  try:
    gpu = 'GPU-%s' % uuid.UUID(bytes=bytes(torch.cuda.get_device_properties(device).uuid.bytes))
    r = subprocess.run(['nvidia-smi', '-i', gpu, '--query-gpu=' + ','.join(fields), '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30)
    values = [v.strip() for v in r.stdout.strip().split(',')]
    if r.returncode or len(values) != len(fields):
      raise RuntimeError((r.stdout + r.stderr).strip() or 'exit status %d' % r.returncode)
    return values
  except Exception as e:
    return ['unknown (%s)' % e] * len(fields)


def card(device=None):
  """Name, power limit and maximum SM clock of CUDA device ``device`` (default: the current one)."""
  name, power_limit, max_sm_clock = nvidia_smi(('name', 'power.limit', 'clocks.max.sm'), device)
  return {'name': name, 'power_limit': power_limit, 'max_sm_clock': max_sm_clock}


def step_ms(fn, items, warmup):
  """Milliseconds of fn(item) for each item after the first ``warmup``: CUDA events on the current stream around
  the call and a device synchronise after it, so every step starts on an idle device."""
  ms = []
  for i, item in enumerate(items):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn(item)
    e1.record()
    torch.cuda.synchronize()
    if i >= warmup:
      ms.append(e0.elapsed_time(e1))
  return ms


def back_to_back_ms(fn, items, warmup):
  """Milliseconds of fn(item) for each item after the first ``warmup``, with the steps run back to back as in the
  training loop: one event on the current stream at each step boundary and one synchronise of that stream after
  the last step.  Nothing synchronises the device in between, so the copies a staged image bank issues after a
  step overlap the next step as they do in training."""
  marks = [torch.cuda.Event(enable_timing=True)]
  marks[0].record()
  for item in items:
    fn(item)
    marks.append(torch.cuda.Event(enable_timing=True))
    marks[-1].record()
  torch.cuda.current_stream().synchronize()
  return [a.elapsed_time(b) for a, b in zip(marks[warmup:], marks[warmup + 1:])]


def summary(ms):
  """The median, min and max of step times, as the tools print them."""
  return {'ms_per_step_median': round(float(np.median(ms)), 3), 'ms_per_step_min': round(float(np.min(ms)), 3),
          'ms_per_step_max': round(float(np.max(ms)), 3)}


def spawn_ranks(fn, world, backend):
  """Run fn(rank, world) in ``world`` spawned processes joined in one ``backend`` process group on this host, and
  return what rank 0's call returned (through a JSON file).  Rank r uses GPU r under NCCL and GPU 0 otherwise.
  ``fn`` must be picklable: a module-level function or a functools.partial of one."""
  import torch.multiprocessing as mp
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  port = s.getsockname()[1]
  s.close()
  with tempfile.TemporaryDirectory() as tmp:
    out = os.path.join(tmp, 'rank0.json')
    mp.spawn(_rank, args=(fn, world, backend, port, out), nprocs=world, join=True)
    with open(out) as f:
      return json.load(f)


def _rank(rank, fn, world, backend, port, out):
  import torch.distributed as dist
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(rank if backend == 'nccl' else 0)
  dist.init_process_group(backend, rank=rank, world_size=world)
  try:
    result = fn(rank, world)
    if rank == 0:
      with open(out, 'w') as f:
        json.dump(result, f)
  finally:
    dist.destroy_process_group()
