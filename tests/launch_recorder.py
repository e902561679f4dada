"""Records the launches a train step makes through multinerf_b200.ops, for the GPU tests that check each launch (or
each stage the model composes from them) against an fp64 reference on the tensors that launch really saw.

`Recorder(ops, names, monkeypatch)` wraps the named ops functions.  Every call becomes a `Call` with `fn`, `args`
(every argument by name, the live objects: compare `data_ptr()`s to find which buffer an operand is), `before` (a
clone of every tensor argument taken before the call) and `after` (clones taken after it, behind a synchronize).
"""
import inspect
import types

import torch


class Recorder:

  def __init__(self, ops_, names, monkeypatch):
    self.calls = []
    for name in names:
      fn = getattr(ops_, name)
      monkeypatch.setattr(ops_, name, self._wrap(name, fn, inspect.signature(fn)))

  def _wrap(self, name, fn, sig):
    def call(*a, **kw):
      args = sig.bind(*a, **kw).arguments
      before = {k: v.clone() for k, v in args.items() if torch.is_tensor(v)}
      r = fn(*a, **kw)
      torch.cuda.synchronize()
      after = {k: v.clone() for k, v in args.items() if torch.is_tensor(v)}
      self.calls.append(types.SimpleNamespace(fn=name, args=args, before=before, after=after))
      return r
    return call

  def of(self, fn, **ptrs):
    """The calls of `fn` whose named tensor arguments start at the given tensors' addresses."""
    return [c for c in self.calls if c.fn == fn and
            all(torch.is_tensor(c.args.get(k)) and c.args[k].data_ptr() == t.data_ptr() for k, t in ptrs.items())]
