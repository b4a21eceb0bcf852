"""`pip install --no-build-isolation .` — runs `make` (g++ + nvcc for sm_90a; no GPU needed) and ships the three plugin
variants inside the package (bagua_net_b200/lib/).  Working from a checkout needs none of this: the library is built in
the tree on first use (bagua_net_b200._build) and `make install PREFIX=...` copies the plugin for NCCL alone.
Counterpart of the reference's `make && make install` (reference: cc/Makefile, README.md:32-45)."""
import os
import subprocess

from setuptools import setup
from setuptools.command.build_py import build_py

ROOT = os.path.dirname(os.path.abspath(__file__))


class BuildWithNative(build_py):
    def run(self):
        jobs = str(min(16, os.cpu_count() or 4))
        subprocess.run(["make", "-C", ROOT, "-j" + jobs], check=True)
        super().run()


setup(cmdclass={"build_py": BuildWithNative})
