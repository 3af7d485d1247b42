"""`pip install -e .` / `python setup.py build_ext --inplace`: the native code is built by build.py (ninja + g++ +
nvcc for sm_90a) into blackbird_b200/_bb*.so and bin/; setuptools only packages the result."""
import os
import subprocess
import sys

from setuptools import setup
from setuptools.command.build_py import build_py


class BuildNative(build_py):
    def run(self):
        root = os.path.dirname(os.path.abspath(__file__))
        subprocess.check_call([sys.executable, os.path.join(root, "build.py")], cwd=root)
        super().run()


setup(cmdclass={"build_py": BuildNative})
