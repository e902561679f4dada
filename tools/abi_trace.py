"""Records the sequence of C-ABI calls (`mnrf_*`) that one train step and one render call make, without a GPU.

`lib.load` is replaced by a fake library that records every call and returns 0, and `lib.ptr` by one that returns
the tensor's address and keeps the tensor alive, so that the CPU allocator cannot hand a freed address to a later
tensor and make the trace depend on the run.  Each model is built on the CPU.  Every call is recorded with its
symbol, its scalar arguments and its ctypes descriptors expanded field by field; pointers, in the arguments and
inside descriptors, are numbered in order of first appearance.  Two checkouts that make the same kernel launches,
in the same order, on the same buffers and with the same descriptors give byte-identical traces:

    python tools/abi_trace.py --root /path/to/other/checkout --out other.json
    python tools/abi_trace.py --out this.json
    cmp other.json this.json
"""
import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from abi_record import _bundles, run_case  # noqa: E402  (the recorder the launch-coverage audit shares)


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
  ap.add_argument('--root', default=ROOT, help='checkout whose multinerf_b200 package is traced')
  ap.add_argument('--out', required=True, help='JSON trace to write')
  ap.add_argument('--cases', default='', help='comma-separated subset of the case names')
  args = ap.parse_args()
  sys.path.insert(0, os.path.abspath(args.root))
  from multinerf_b200 import configs, lib, models, train_utils, utils
  pkg = (lib, models, train_utils, utils)
  want = set(filter(None, args.cases.split(',')))
  trace = {}
  for name, fn, env in _bundles(configs):
    if want and name not in want:
      continue
    try:
      trace[name] = run_case(pkg, fn, env)
    except Exception as e:
      raise RuntimeError(f'case {name}') from e
  text = json.dumps(trace, sort_keys=True, separators=(',', ':'))
  with open(args.out, 'w') as fh:
    fh.write(text)
  for name, case in trace.items():
    print(f'{name:32s} train {case["train_calls"]:4d}  render {case["render_calls"]:4d}')
  print('sha1', hashlib.sha1(text.encode()).hexdigest())


if __name__ == '__main__':
  main()
