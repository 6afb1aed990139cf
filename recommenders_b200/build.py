"""Builds recommenders_b200/libtfrs_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m recommenders_b200.build [--force] [--verbose]

The .so and the object files are build products (git-ignored); __graft_entry__.build() runs this.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "csrc", "build")
LIB = os.path.join(HERE, "libtfrs_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
    "-DTFRS_BUILD",
]


def _nvcc() -> str:
  for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
    if c and os.path.exists(c):
      return c
  raise RuntimeError("nvcc not found; libtfrs_b200.so cannot be built")


def _sources():
  return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest() -> str:
  h = hashlib.sha256()
  files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))]
  files.append(os.path.join(HERE, "..", "include", "tfrs_b200.h"))
  for f in files:
    with open(f, "rb") as fh:
      h.update(f.encode()); h.update(fh.read())
  h.update(" ".join(NVCC_FLAGS).encode())
  return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
  stamp = os.path.join(OBJ, "stamp")
  dig = _digest()
  if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
    return LIB
  os.makedirs(OBJ, exist_ok=True)
  nvcc = _nvcc()
  # nvcc's host compiler: prefer the system g++ when there is one
  ccbin = ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []

  def compile_one(src):
    obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
    cmd = [nvcc, *ccbin, *NVCC_FLAGS, "-c", src, "-o", obj]
    if verbose:
      cmd.insert(1, "-Xptxas"); cmd.insert(2, "-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
      raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
      sys.stderr.write(r.stderr)
    return obj

  with cf.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 2)) as ex:
    objs = list(ex.map(compile_one, _sources()))
  cmd = [nvcc, *ccbin, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs,
         "-Xcompiler", "-fPIC", "-cudart", "static", "-ldl"]
  r = subprocess.run(cmd, capture_output=True, text=True)
  if r.returncode != 0:
    raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
  with open(stamp, "w") as fh:
    fh.write(dig)
  return LIB


if __name__ == "__main__":
  print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
