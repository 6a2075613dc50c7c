r"""Kubernetes launcher for H100 node pools (ref `lingvo/tools/gke_launch.py`, which deploys a
TPU trainer job, GPU decoder jobs and TensorBoard on GKE from one command line).

Same workflow, H100 shape:

  * **trainer** — an Indexed `Job` with one pod per node, every pod requesting all the node's
    GPUs (`nvidia.com/gpu: 8`) and running `torchrun --nnodes=N --nproc-per-node=8 -m
    lingvo_b200.trainer …`; pods find each other through a headless `Service` (rendezvous on
    pod 0), `/dev/shm` is a memory-backed volume (NCCL / CUDA IPC symmetric memory need it),
    and `hostIPC` is on so that peer-memory handles can be exchanged inside the node;
  * **decoder** / **evaler** — `Deployment`s with `--decoder_gpus` GPUs that follow the
    checkpoints in `--logdir` (`--job=decoder_<split>` / `evaler_<split>`);
  * **tensorboard** — a `Deployment` + `LoadBalancer` `Service` on the event files.

    python -m lingvo_b200.tools.gke_launch --name=moe --model=lm.synthetic_packed_input.MoELm8E \
        --image=registry/lingvo_b200:tag --logdir=/mnt/logs/moe --nodes=2 \
        [--build=. --base_image=…] [--cluster=ctx] up|down|reload|print [trainer|decoder|evaler|tensorboard|all]

`print` writes the manifests to a temp dir and prints them; `up` / `down` call
`kubectl create|delete -f`; `reload` = down + up; `--build=<dir>` first builds (and pushes) the
image from `docker/Dockerfile`. Nothing here needs a cluster to be *generated*, so the
manifests are unit-tested.
"""

from __future__ import annotations

import argparse
import datetime
import os
import shlex
import subprocess
import sys
import tempfile

import yaml

ACTIONS = ('up', 'down', 'reload', 'print')
TARGETS = ('trainer', 'decoder', 'evaler', 'tensorboard')


def ParseArgs(argv=None):
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument('--name', required=True, help='Base name of the experiment.')
  ap.add_argument('--model', required=True, help='Name of the registered model.')
  ap.add_argument('--image', required=True, help='Container image to run.')
  ap.add_argument('--logdir', required=True, help='Shared log directory (mounted volume).')
  ap.add_argument('--nodes', type=int, default=1, help='Trainer nodes (pods).')
  ap.add_argument('--gpus_per_node', type=int, default=8, help='GPUs (processes) per node.')
  ap.add_argument('--gpu_type', default='nvidia-b200', help='Node-selector accelerator label.')
  ap.add_argument('--shm_size', default='64Gi', help='Size of the memory-backed /dev/shm.')
  ap.add_argument('--logdir_pvc', default='', help='PersistentVolumeClaim holding --logdir '
                  '(empty: hostPath).')
  ap.add_argument('--decoder', default='dev', help='Comma-separated dataset splits to decode.')
  ap.add_argument('--evaler', default='dev', help='Comma-separated dataset splits to evaluate.')
  ap.add_argument('--decoder_gpus', type=int, default=1, help='GPUs per decoder / evaler pod.')
  ap.add_argument('--decoder_ram', default='24G', help='Memory request of decoder pods.')
  ap.add_argument('--tensorboard_port', type=int, default=6006)
  ap.add_argument('--mode', default='sync', choices=('sync', 'async'))
  ap.add_argument('--extra_args', default='', help='Extra trainer flags, verbatim.')
  ap.add_argument('--extra_envs', default='', help='Comma-separated K=V pairs for every pod.')
  ap.add_argument('--cluster', default='', help='kubectl context / cluster to target.')
  ap.add_argument('--build', default='', help='Build the image from this source directory first.')
  ap.add_argument('--base_image', default='nvidia/cuda:12.9.0-devel-ubuntu24.04')
  ap.add_argument('--master_port', type=int, default=29500)
  ap.add_argument('action', choices=ACTIONS)
  ap.add_argument('target', nargs='?', default='all', choices=TARGETS + ('all',))
  return ap.parse_args(argv)


# ------------------------------------------------------------------------ manifests --
def _Env(args, extra=()):
  env = [{'name': 'NCCL_DEBUG', 'value': 'WARN'}, {'name': 'PYTHONUNBUFFERED', 'value': '1'}]
  for kv in filter(None, args.extra_envs.split(',')):
    k, _, v = kv.partition('=')
    env.append({'name': k, 'value': v})
  return env + list(extra)


def _Volumes(args):
  vols = [{'name': 'dshm', 'emptyDir': {'medium': 'Memory', 'sizeLimit': args.shm_size}}]
  if args.logdir_pvc:
    vols.append({'name': 'logdir', 'persistentVolumeClaim': {'claimName': args.logdir_pvc}})
  else:
    vols.append({'name': 'logdir', 'hostPath': {'path': args.logdir, 'type': 'DirectoryOrCreate'}})
  mounts = [{'name': 'dshm', 'mountPath': '/dev/shm'},
            {'name': 'logdir', 'mountPath': args.logdir}]
  return vols, mounts


def _GpuResources(n, memory=None):
  lim = {'nvidia.com/gpu': int(n)}
  res = {'limits': dict(lim)}
  if memory:
    res['requests'] = {'memory': memory}
  return res


def TrainerCommand(args):
  """The per-pod command: torchrun with pod 0 of the headless service as rendezvous."""
  master = '%s-trainer-0.%s-trainer' % (args.name, args.name)
  cmd = ['python3', '-m', 'torch.distributed.run', '--nnodes=%d' % args.nodes,
         '--nproc-per-node=%d' % args.gpus_per_node, '--node-rank=$(JOB_COMPLETION_INDEX)',
         '--master-addr=%s' % (master if args.nodes > 1 else '127.0.0.1'),
         '--master-port=%d' % args.master_port, '-m', 'lingvo_b200.trainer',
         '--model=%s' % args.model, '--logdir=%s' % args.logdir, '--mode=%s' % args.mode,
         '--job=trainer_client', '--worker_gpus=%d' % args.gpus_per_node,
         '--worker_replicas=%d' % args.nodes]
  return cmd + shlex.split(args.extra_args)


def TrainerManifests(args):
  vols, mounts = _Volumes(args)
  name = '%s-trainer' % args.name
  service = {
      'apiVersion': 'v1', 'kind': 'Service', 'metadata': {'name': name},
      'spec': {'clusterIP': 'None', 'selector': {'job-name': name},
               'ports': [{'name': 'rdzv', 'port': args.master_port}]}}
  pod = {
      'metadata': {'labels': {'app': name}},
      'spec': {
          'restartPolicy': 'Never', 'subdomain': name, 'hostIPC': True,
          'nodeSelector': {'cloud.google.com/gke-accelerator': args.gpu_type},
          'tolerations': [{'key': 'nvidia.com/gpu', 'operator': 'Exists',
                           'effect': 'NoSchedule'}],
          'volumes': vols,
          'containers': [{
              'name': 'trainer', 'image': args.image,
              'command': ['/bin/bash', '-c', ' '.join(TrainerCommand(args))],
              'env': _Env(args), 'volumeMounts': mounts,
              'resources': _GpuResources(args.gpus_per_node),
              'securityContext': {'capabilities': {'add': ['IPC_LOCK']}}}]}}
  job = {
      'apiVersion': 'batch/v1', 'kind': 'Job', 'metadata': {'name': name},
      'spec': {'completions': args.nodes, 'parallelism': args.nodes,
               'completionMode': 'Indexed', 'backoffLimit': 0, 'template': pod}}
  return [service, job]


def FollowerManifest(args, kind, split):
  """A decoder / evaler deployment following the checkpoints in --logdir."""
  assert kind in ('decoder', 'evaler')
  vols, mounts = _Volumes(args)
  name = '%s-%s-%s' % (args.name, kind, split)
  cmd = ['python3', '-m', 'lingvo_b200.trainer', '--model=%s' % args.model,
         '--logdir=%s' % args.logdir, '--job=%s_%s' % (kind, split), '--mode=sync',
         '--%s_gpus=%d' % (kind, args.decoder_gpus)]
  return {
      'apiVersion': 'apps/v1', 'kind': 'Deployment', 'metadata': {'name': name},
      'spec': {'replicas': 1, 'selector': {'matchLabels': {'app': name}},
               'template': {
                   'metadata': {'labels': {'app': name}},
                   'spec': {
                       'nodeSelector': ({'cloud.google.com/gke-accelerator': args.gpu_type}
                                        if args.decoder_gpus else {}),
                       'volumes': vols,
                       'containers': [{
                           'name': kind, 'image': args.image, 'command': cmd,
                           'env': _Env(args), 'volumeMounts': mounts,
                           'resources': _GpuResources(args.decoder_gpus, args.decoder_ram)
                           if args.decoder_gpus else {'requests': {'memory': args.decoder_ram}},
                       }]}}}}


def TensorboardManifests(args):
  vols, mounts = _Volumes(args)
  name = '%s-tensorboard' % args.name
  dep = {
      'apiVersion': 'apps/v1', 'kind': 'Deployment', 'metadata': {'name': name},
      'spec': {'replicas': 1, 'selector': {'matchLabels': {'app': name}},
               'template': {'metadata': {'labels': {'app': name}},
                            'spec': {'volumes': vols[1:], 'containers': [{
                                'name': 'tensorboard', 'image': args.image,
                                'command': ['tensorboard', '--logdir=%s' % args.logdir,
                                            '--port=%d' % args.tensorboard_port,
                                            '--bind_all'],
                                'ports': [{'containerPort': args.tensorboard_port}],
                                'volumeMounts': mounts[1:]}]}}}}
  svc = {'apiVersion': 'v1', 'kind': 'Service', 'metadata': {'name': name},
         'spec': {'type': 'LoadBalancer', 'selector': {'app': name},
                  'ports': [{'port': 80, 'targetPort': args.tensorboard_port}]}}
  return [dep, svc]


def BuildManifests(args, targets):
  out = {}
  if 'trainer' in targets:
    out['trainer.yaml'] = TrainerManifests(args)
  for kind in ('decoder', 'evaler'):
    if kind in targets:
      splits = [s for s in getattr(args, kind).split(',') if s]
      if splits:
        out['%s.yaml' % kind] = [FollowerManifest(args, kind, s) for s in splits]
  if 'tensorboard' in targets:
    out['tensorboard.yaml'] = TensorboardManifests(args)
  return out


# ------------------------------------------------------------------------- actions --
def BuildDockerImage(image, base_image, code_directory, run=subprocess.check_call):
  """docker build (from docker/Dockerfile with BASE_IMAGE) + push (ref :278)."""
  dockerfile = os.path.join(code_directory, 'docker', 'Dockerfile')
  run(['docker', 'build', '-t', image, '-f', dockerfile, '--build-arg',
       'BASE_IMAGE=%s' % base_image, code_directory])
  run(['docker', 'push', image])
  return image


def _Kubectl(verb, path, cluster, run):
  cmd = ['kubectl', verb, '-f', path]
  if cluster:
    cmd += ['--context', cluster]
  print('Running: %s' % ' '.join(cmd))
  return run(cmd)


def Main(argv=None, run=subprocess.call):
  args = ParseArgs(argv)
  targets = list(TARGETS) if args.target == 'all' else [args.target]
  actions = ['down', 'up'] if args.action == 'reload' else [args.action]
  image = args.image
  if 'up' in actions and args.build:
    if ':' not in image.rsplit('/', 1)[-1]:
      image += ':%s' % datetime.datetime.now().strftime('%Y-%m-%d_%H-%M-%S')
    args.image = BuildDockerImage(image, args.base_image, args.build, run=run)
  root = tempfile.mkdtemp(prefix=args.name + '-')
  print('Writing out yaml configs to %s' % root)
  paths = {}
  for fname, docs in BuildManifests(args, targets).items():
    paths[fname] = os.path.join(root, fname)
    with open(paths[fname], 'w') as f:
      yaml.safe_dump_all(docs, f, sort_keys=False)
  rc = 0
  for action in actions:
    for fname, path in paths.items():
      if action == 'print':
        print('# ---- %s' % fname)
        print(open(path).read())
      else:
        rc = _Kubectl({'up': 'create', 'down': 'delete'}[action], path, args.cluster, run) or rc
  return rc, paths


if __name__ == '__main__':
  sys.exit(Main()[0])
