"""pip install .  -- packages the hyphenated source directory as the importable package ``qsa_b200`` together with the
C ABI: libsa_b200.so (built here with nvcc for sm_90a if it is not there yet) and the headers (qsa_b200/include/*.h).
A source checkout needs none of this: ``qsa_b200/__init__.py`` there is a path shim onto the same directory."""
import os
import shutil
import subprocess

from setuptools import setup
from setuptools.command.build_py import build_py

ROOT = os.path.dirname(os.path.abspath(__file__))
PKG_DIR = "quickstart-streaming-agents_b200"


class BuildWithNative(build_py):
    def run(self):
        so = os.path.join(ROOT, PKG_DIR, "libsa_b200.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-C", os.path.join(ROOT, PKG_DIR, "csrc")])
        super().run()
        dst = os.path.join(self.build_lib, "qsa_b200")
        shutil.copy2(so, os.path.join(dst, "libsa_b200.so"))
        os.makedirs(os.path.join(dst, "include"), exist_ok=True)
        for h in ("sa_api.h", "sa_wire.h"):
            shutil.copy2(os.path.join(ROOT, "include", h), os.path.join(dst, "include", h))


SUB = ["embed", "pipeline", "transport", "wire"]
setup(
    packages=["qsa_b200"] + [f"qsa_b200.{s}" for s in SUB] + ["scripts"],
    package_dir={"qsa_b200": PKG_DIR, **{f"qsa_b200.{s}": f"{PKG_DIR}/{s}" for s in SUB}, "scripts": "scripts"},
    cmdclass={"build_py": BuildWithNative},
)
