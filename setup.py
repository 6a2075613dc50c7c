"""Packaging (ref `pip_package/`): `pip install .` builds the sm_90a kernel extension and
the host runtime in-tree through `lingvo_b200.ops.build`, then installs the package."""

import os
import subprocess
import sys

from setuptools import find_packages
from setuptools import setup
from setuptools.command.build_py import build_py


class BuildWithExtensions(build_py):

  def run(self):
    root = os.path.dirname(os.path.abspath(__file__))
    subprocess.check_call([sys.executable, '-c', 'import __graft_entry__ as g; g.build()'],
                          cwd=root)
    super().run()


setup(
    name='lingvo_b200',
    version='0.2.0',
    description='H100-native (sm_90a) sequence-modelling framework with the capabilities of Lingvo',
    packages=find_packages(include=['lingvo_b200', 'lingvo_b200.*']),
    package_data={'lingvo_b200.ops': ['*.so', 'csrc/*', 'csrc_host/*']},
    python_requires='>=3.10',
    install_requires=['torch>=2.4', 'numpy', 'pyyaml', 'absl-py'],
    entry_points={'console_scripts': ['lingvo_b200_trainer = lingvo_b200.trainer:main_cli']},
    cmdclass={'build_py': BuildWithExtensions},
)
