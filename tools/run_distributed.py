#!/usr/bin/env python
"""Local multi-process launcher (ref `docker/run_distributed.py`: a docker fleet of
`worker×3, controller, trainer_client` (sync) or `trainer×3, ps×2, controller` (async)).

On H100 the topology is one process per GPU: a *trainer* job of N ranks under
`torch.distributed.run`, plus optional *evaler* / *decoder* side jobs that poll the same
log dir (they need no rendezvous with the trainer).

  tools/run_distributed.py --model=lm.synthetic_packed_input.MoELm8E --logdir=/tmp/moe \
      --gpus=8 [--evaler_dev] [--decoder_dev] [--dry_run]
"""

import argparse
import os
import shlex
import subprocess
import sys


def Commands(a):
  base = [sys.executable, '-m', 'lingvo_b200.trainer', '--model=' + a.model,
          '--logdir=' + a.logdir, '--mode=sync']
  base += shlex.split(a.extra_flags)
  cmds = []
  if a.gpus > 1:
    cmds.append(('trainer', [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1',
                             '--nproc-per-node=%d' % a.gpus, '--master-addr=127.0.0.1',
                             '--master-port=%d' % a.port, '-m', 'lingvo_b200.trainer'] +
                 base[3:] + ['--job=trainer_client']))
  else:
    cmds.append(('trainer', base + ['--job=controller,trainer_client']))
  if a.evaler_dev:
    cmds.append(('evaler_dev', base + ['--job=evaler_dev']))
  if a.decoder_dev:
    cmds.append(('decoder_dev', base + ['--job=decoder_dev']))
  return cmds


def main(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--model', required=True)
  ap.add_argument('--logdir', required=True)
  ap.add_argument('--gpus', type=int, default=1)
  ap.add_argument('--port', type=int, default=29500)
  ap.add_argument('--evaler_dev', action='store_true')
  ap.add_argument('--decoder_dev', action='store_true')
  ap.add_argument('--extra_flags', default='')
  ap.add_argument('--dry_run', action='store_true')
  a = ap.parse_args(argv)
  cmds = Commands(a)
  if a.dry_run:
    for name, c in cmds:
      print('%-12s %s' % (name, ' '.join(shlex.quote(x) for x in c)))
    return 0
  os.makedirs(a.logdir, exist_ok=True)
  procs = []
  for name, c in cmds:
    log = open(os.path.join(a.logdir, name + '.log'), 'w')
    env = dict(os.environ)
    if name != 'trainer':                      # side jobs share GPU 0 unless told otherwise
      env.setdefault('CUDA_VISIBLE_DEVICES', '0')
    procs.append((name, subprocess.Popen(c, stdout=log, stderr=subprocess.STDOUT, env=env)))   # noqa: S603
  rc = procs[0][1].wait()
  for name, p in procs[1:]:
    p.terminate()
  return rc


if __name__ == '__main__':
  sys.exit(main())
