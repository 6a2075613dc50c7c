"""Builds the `lingvo_b200` wheel (ref `pip_package/build.sh`, `build_pip_pkg.sh`).

    python pip_package/build_pip_pkg.py [--out dist] [--skip-native] [--plat manylinux_2_34_x86_64]

Steps: (1) compile the native extensions in-tree (`__graft_entry__.build()`: nvcc for
sm_90a → `_C.so`, g++ → `_H.so`); (2) stage the package + the built `.so` files;
(3) write the wheel by hand (a wheel is a zip with `WHEEL` / `METADATA` / `RECORD`), tagged
for this interpreter and platform because it carries compiled code. No network and no
`build` / `wheel` front-end is needed, which is what the offline image requires.
"""

import argparse
import base64
import hashlib
import os
import sys
import sysconfig
import zipfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME, VERSION = 'lingvo_b200', '0.2.0'


def _Files(skip_native):
  keep_ext = ('.py', '.cu', '.cuh', '.cpp', '.h', '.hpp', '.txt', '.md', '.proto')
  for base, dirs, files in os.walk(os.path.join(ROOT, NAME)):
    dirs[:] = [d for d in dirs if d not in ('__pycache__', '_obj', 'build')]
    for f in files:
      if f.endswith(keep_ext) or (f.endswith('.so') and not skip_native):
        full = os.path.join(base, f)
        yield full, os.path.relpath(full, ROOT)


def _Record(data: bytes):
  digest = base64.urlsafe_b64encode(hashlib.sha256(data).digest()).rstrip(b'=').decode()
  return 'sha256=%s,%d' % (digest, len(data))


def BuildWheel(out_dir, skip_native=False, plat=None):
  if not skip_native:
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g   # pylint: disable=g-import-not-at-top,import-error
    g.build()
  py = 'cp%d%d' % sys.version_info[:2]
  plat = plat or sysconfig.get_platform().replace('-', '_').replace('.', '_')
  tag = '%s-%s-%s' % (py, py, plat) if not skip_native else 'py3-none-any'
  os.makedirs(out_dir, exist_ok=True)
  path = os.path.join(out_dir, '%s-%s-%s.whl' % (NAME, VERSION, tag))
  dist_info = '%s-%s.dist-info' % (NAME, VERSION)
  records = []
  with zipfile.ZipFile(path, 'w', zipfile.ZIP_DEFLATED) as z:
    def Add(arc, data):
      z.writestr(arc, data)
      records.append('%s,%s' % (arc, _Record(data)))
    for full, arc in sorted(_Files(skip_native)):
      with open(full, 'rb') as f:
        Add(arc, f.read())
    meta = ('Metadata-Version: 2.1\nName: %s\nVersion: %s\nSummary: H100-native (sm_90a) '
            'sequence-modelling framework with the capabilities of Lingvo\n'
            'Requires-Python: >=3.10\nRequires-Dist: torch>=2.4\nRequires-Dist: numpy\n'
            'Requires-Dist: pyyaml\nRequires-Dist: absl-py\n' % (NAME, VERSION))
    Add('%s/METADATA' % dist_info, meta.encode())
    Add('%s/WHEEL' % dist_info, ('Wheel-Version: 1.0\nGenerator: lingvo_b200-build_pip_pkg\n'
                                 'Root-Is-Purelib: %s\nTag: %s\n' %
                                 ('true' if skip_native else 'false', tag)).encode())
    Add('%s/entry_points.txt' % dist_info,
        b'[console_scripts]\nlingvo_b200_trainer = lingvo_b200.trainer:main_cli\n')
    Add('%s/top_level.txt' % dist_info, (NAME + '\n').encode())
    records.append('%s/RECORD,,' % dist_info)
    z.writestr('%s/RECORD' % dist_info, '\n'.join(records) + '\n')
  return path


if __name__ == '__main__':
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=os.path.join(ROOT, 'dist'))
  ap.add_argument('--skip-native', action='store_true')
  ap.add_argument('--plat', default=None)
  a = ap.parse_args()
  print(BuildWheel(a.out, a.skip_native, a.plat))
