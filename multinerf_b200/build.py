"""Builds multinerf_b200/libmnrf_b200.so (sm_90a) in-tree with nvcc.  No GPU needed."""
import concurrent.futures
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, '..', 'build', 'obj')
LIB = os.path.join(HERE, 'libmnrf_b200.so')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
COMMON = ['-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']
# The per-ray geometry/compositing kernels are compiled without FMA contraction so that their
# fp32 rounding follows the reference's unfused elementwise graph (tight oracle parity); the
# GEMM and reduction kernels keep FMA.
SOURCES = {
    'lib.cu': [], 'sampling.cu': ['-fmad=false'], 'encode.cu': ['-fmad=false'],
    'composite.cu': ['-fmad=false'], 'heads.cu': [], 'gemm_tc.cu': [], 'gemm_tc_act.cu': [], 'chain.cu': [],
    'gemm_ref.cu': [],
    'refnerf.cu': [], 'camera.cu': ['-fmad=false'], 'robust.cu': ['-fmad=false'], 'mesh.cu': ['-fmad=false'],
    'mesh_trace.cu': ['-fmad=false'],
}


def _nvcc():
  for cand in [os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc']:
    if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
      return cand
  raise RuntimeError('nvcc not found')


# sources a unit includes besides the shared headers
INCLUDES = {'gemm_tc_act.cu': ['gemm_tc.cu'], 'mesh.cu': ['mc_tables.cuh', 'camera.cuh', 'contract.cuh'],
            'camera.cu': ['camera.cuh'], 'encode.cu': ['contract.cuh']}


def _stamp(path, flags):
  h = hashlib.sha1()
  extra = [os.path.join(CSRC, f) for f in INCLUDES.get(os.path.basename(path), [])]
  for p in [path] + extra + [os.path.join(CSRC, 'common.cuh'), os.path.join(CSRC, 'tc_common.cuh'),
            os.path.join(CSRC, 'wgmma.cuh'), os.path.join(HERE, '..', 'include', 'mnrf.h')]:
    with open(p, 'rb') as f:
      h.update(f.read())
  h.update(' '.join(flags).encode())
  return h.hexdigest()


def _compile(name, flags, verbose):
  src = os.path.join(CSRC, name)
  obj = os.path.join(OBJ, name.replace('.cu', '.o'))
  stamp_file = obj + '.stamp'
  stamp = _stamp(src, flags)
  if os.path.exists(obj) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
    return obj, False
  cmd = [_nvcc()] + ARCH + COMMON + flags + ['-c', src, '-o', obj]
  if verbose:
    print(' '.join(cmd), flush=True)
  subprocess.run(cmd, check=True)
  with open(stamp_file, 'w') as f:
    f.write(stamp)
  return obj, True


def build(verbose=False, force=False):
  os.makedirs(OBJ, exist_ok=True)
  if force:
    for f in os.listdir(OBJ):
      os.remove(os.path.join(OBJ, f))
  with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
    results = list(ex.map(lambda kv: _compile(kv[0], kv[1], verbose), SOURCES.items()))
  objs = [r[0] for r in results]
  if any(r[1] for r in results) or not os.path.exists(LIB):
    cmd = [_nvcc()] + ARCH + ['-shared', '-o', LIB] + objs
    if verbose:
      print(' '.join(cmd), flush=True)
    subprocess.run(cmd, check=True)
  return LIB


if __name__ == '__main__':
  print(build(verbose=True, force='--force' in sys.argv))
