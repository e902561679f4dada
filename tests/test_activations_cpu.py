"""CPU tests of the Dense-layer activations (MLP.net_activation): which activation each MLP plan runs, the same layer
table for every activation, the config errors that name their field, and the C entry points of the smooth
activations."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = ('relu', 'softplus', 'silu')     # what models.Model builds its plans for


def test_smooth_activation_keeps_the_layer_table():
  # blender_256.gin: 835,205 parameters (scripts/generate_tables.ipynb) whatever the activation
  from multinerf_b200 import configs
  from multinerf_b200 import lib as L
  from multinerf_b200.models import MLPPlan
  bb = configs.bundle_blender_256()
  relu = MLPPlan(bb.nerf_mlp, activations=ALL)
  bb.nerf_mlp.net_activation = 'silu'
  silu = MLPPlan(bb.nerf_mlp, activations=ALL)
  assert silu.num_params + MLPPlan(bb.prop_mlp, activations=ALL).num_params == 835205
  assert [(s.name, s.in_dim, s.in_pad, s.out_dim) for s in silu.specs] == \
      [(s.name, s.in_dim, s.in_pad, s.out_dim) for s in relu.specs]
  assert {sp.act for sp in silu.specs if sp.role in ('trunk', 'view')} == {L.ACT_SILU}
  assert {sp.act for sp in relu.specs if sp.role in ('trunk', 'view')} == {L.ACT_RELU}
  # the bare table is the ReLU one: a caller that runs a smooth schedule says so
  with pytest.raises(NotImplementedError, match='net_activation'):
    MLPPlan(bb.nerf_mlp)


@pytest.mark.parametrize('fn,code', [('silu', 'ACT_SILU'), ('softplus', 'ACT_SOFTPLUS'), ('relu', 'ACT_RELU')])
def test_gin_net_activation_sets_plan_activation(fn, code):
  from multinerf_b200 import configs
  from multinerf_b200 import lib as L
  from multinerf_b200.models import MLPPlan
  b = configs.parse_gin(f'NerfMLP.net_activation = @jax.nn.{fn}\n', configs.bundle_blender_256())
  assert b.nerf_mlp.net_activation == fn and b.prop_mlp.net_activation == 'relu'
  assert MLPPlan(b.nerf_mlp, activations=ALL).act == getattr(L, code)
  assert MLPPlan(b.prop_mlp, activations=ALL).act == L.ACT_RELU      # each MLP has its own


@pytest.mark.parametrize('text,field', [('NerfMLP.net_activation = @jnp.exp', 'net_activation'),
                                        ('NerfMLP.density_activation = @jax.nn.relu', 'density_activation'),
                                        ('NerfMLP.roughness_activation = @jax.nn.relu', 'roughness_activation')])
def test_unsupported_activation_names_its_field(text, field):
  from multinerf_b200 import configs
  from multinerf_b200.models import MLPPlan
  b = configs.parse_gin(text + '\n', configs.bundle_blender_256())
  with pytest.raises(NotImplementedError, match=field):
    MLPPlan(b.nerf_mlp, activations=ALL)


def test_smooth_activations_run_through_the_base_entry_points():
  from multinerf_b200 import lib
  if not os.path.exists(lib.LIB_PATH):
    from multinerf_b200 import build
    build.build()
  l = lib.load()
  for name in ('mnrf_gemm', 'mnrf_head_bwd', 'mnrf_act_tangent_bwd'):
    assert name in lib.EXPORTED and hasattr(l, name)
  # the smooth activations run through the base entries, which take the pre-activation z and its pitch
  header = open(os.path.join(ROOT, 'include', 'mnrf.h')).read()
  for name in ('mnrf_gemm', 'mnrf_head_bwd'):
    decl = re.search(r'\b' + name + r'\(([^;]*)\);', header)
    assert decl and 'mnrf_bf16* z' in decl.group(1) and 'int64_t ldz' in decl.group(1), name
  for name in ('mnrf_gemm_act', 'mnrf_head_bwd_act'):
    assert name not in lib.EXPORTED and not hasattr(l, name)
  assert (lib.ACT_NONE, lib.ACT_RELU, lib.ACT_SOFTPLUS, lib.ACT_SILU) == (0, 1, 2, 3)
