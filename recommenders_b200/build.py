"""Builds recommenders_b200/libtfrs_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m recommenders_b200.build [--force] [--verbose]
    python -m recommenders_b200.build --debug-switches VARIANT [--out PATH] [--force] [--verbose]

The .so and the object files are build products (git-ignored); __graft_entry__.build() runs this.

--debug-switches builds a separate library with the TFRS_DEBUG_SWITCHES A/B switches compiled in (DEBUG_VARIANTS below),
by default recommenders_b200/debug/libtfrs_b200_<VARIANT>.so, for tools/filter_probe.py to load through TFRS_B200_LIB.  The
product library, its objects and its build digest are left alone.
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

# ablations of the top-K filter pass (csrc/topk_tc.cu); "full" is the product code with the runtime debug switches
DEBUG_VARIANTS = {
    "full": [],
    "no-emit": ["-DTFRS_FILTER_ABLATION=1"],
    "no-epilogue": ["-DTFRS_FILTER_ABLATION=2"],
}


def _nvcc() -> str:
  for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
    if c and os.path.exists(c):
      return c
  raise RuntimeError("nvcc not found; libtfrs_b200.so cannot be built")


def _sources():
  return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(flags) -> str:
  h = hashlib.sha256()
  files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))]
  files.append(os.path.join(HERE, "..", "include", "tfrs_b200.h"))
  for f in files:
    with open(f, "rb") as fh:
      h.update(f.encode()); h.update(fh.read())
  h.update(" ".join(flags).encode())
  return h.hexdigest()


def build(force: bool = False, verbose: bool = False, debug_variant: str | None = None, out: str | None = None) -> str:
  if debug_variant is None:
    flags, obj_dir, lib = NVCC_FLAGS, OBJ, LIB
  else:
    flags = NVCC_FLAGS + ["-DTFRS_DEBUG_SWITCHES", *DEBUG_VARIANTS[debug_variant]]
    obj_dir = os.path.join(OBJ, "debug-" + debug_variant)
    lib = os.path.abspath(out) if out else os.path.join(HERE, "debug", f"libtfrs_b200_{debug_variant}.so")
    os.makedirs(os.path.dirname(lib), exist_ok=True)
  stamp = os.path.join(obj_dir, "stamp")
  dig = _digest(flags)
  if not force and os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == dig:
    return lib
  os.makedirs(obj_dir, exist_ok=True)
  nvcc = _nvcc()
  # nvcc's host compiler: prefer the system g++ when there is one
  ccbin = ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []

  def compile_one(src):
    obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o")
    cmd = [nvcc, *ccbin, *flags, "-c", src, "-o", obj]
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
  cmd = [nvcc, *ccbin, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib, *objs,
         "-Xcompiler", "-fPIC", "-cudart", "static", "-ldl"]
  r = subprocess.run(cmd, capture_output=True, text=True)
  if r.returncode != 0:
    raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
  with open(stamp, "w") as fh:
    fh.write(dig)
  return lib


if __name__ == "__main__":
  import argparse
  ap = argparse.ArgumentParser()
  ap.add_argument("--force", action="store_true")
  ap.add_argument("--verbose", action="store_true", help="print ptxas -v for every kernel")
  ap.add_argument("--debug-switches", metavar="VARIANT", choices=sorted(DEBUG_VARIANTS), default=None)
  ap.add_argument("--out", default=None, help="library path of a --debug-switches build")
  a = ap.parse_args()
  print(build(force=a.force, verbose=a.verbose, debug_variant=a.debug_switches, out=a.out))
