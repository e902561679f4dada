"""Texture atlases on the GPU: mnrf_mesh_texture_raster against the fp64 restatement of tests/mesh_texture_ref.py at
cell sizes 4, 5 and 11 (uv and texel indices bit for bit, points and normals within per-element bounds, both normal
fallbacks, the ownership invariant on the kernel's own output, the argument checks); the baked texture against
vertex colours on a simplified sphere; extract_mesh and extract_mesh_tsdf with a texture; and the script.  Needs an
H100."""
import os
import sys

import numpy as np
import pytest
import torch

import mesh_texture_ref as R
from test_gpu_mesh import sphere
from test_gpu_mesh_clean import scene  # noqa: F401  (the mini model and its training views)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def mods():
  from multinerf_b200 import lib, mesh, ops
  lib.require_device()
  return lib, ops, mesh


def _special_mesh(seed=0, V=700, F=1000):
  """Random vertices, unit vertex normals and faces, with faces whose vertex normals cancel at weights (1/2, 1/2, 0)
  on both kinds of face (the face's normal is used), zero-area faces (collinear or one point) and faces whose vertex
  normals are all zero."""
  rng = np.random.default_rng(seed)
  v = (rng.normal(size=(V, 3)) * 3).astype(np.float32)
  n = rng.normal(size=(V, 3))
  n = (n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32)
  f = rng.integers(0, V, (F, 3)).astype(np.int32)
  if F < 100:
    return v, f, n
  for face in range(0, 40):                 # opposite normals on corners 0 and 1
    a, b = f[face, 0], f[face, 1]
    n[b] = -n[a]
  v[650:660] = v[649]                        # one point: zero area
  v[640] = [1, 2, 3]
  v[660:670] = v[640] + np.arange(1, 11, dtype=np.float32)[:, None] * np.float32([1, 2, 0.5])  # collinear, exactly
  n[640:670] = 0
  f[40:60] = [[650 + k % 10, 651 + k % 9, 652 + k % 8] for k in range(20)]
  f[60:80] = [[660 + k % 10, 661 + k % 9, 640] for k in range(20)]
  n[f[80:100].ravel()] = 0                  # zero normals: the face's own normal everywhere
  return v, f, n


def _raster(ops, v, f, n, size):
  out = ops.mesh_texture_raster(*(torch.tensor(a, device='cuda') for a in (v, f, n)), size)
  return [t.cpu().numpy() for t in out]


@pytest.mark.parametrize('c', (4, 5, 11))
def test_raster_matches_reference(mods, c):
  _, ops, _ = mods
  v, f, n = _special_mesh()
  # 1000 faces: 500 cells, 23 per row
  size = 23 * c
  assert ops.texture_atlas(len(f), size) == (23, c)
  uv, index, points, normals = _raster(ops, v, f, n, size)
  ruv, rindex, rpoints, rnormals, w, owner = R.raster(v, f, n, size)
  assert uv.dtype == np.float32 and np.array_equal(uv, ruv.astype(np.float32))
  assert index.dtype == np.int32 and np.array_equal(index, rindex)
  assert (np.abs(points - rpoints) <= R.point_bound(v, f, owner)).all()
  bound = R.normal_bound(n, f, owner, w)
  assert (np.abs(normals - rnormals) <= bound).all()
  assert np.allclose(np.linalg.norm(normals, axis=1), 1, atol=4e-7)
  # the fallbacks, where the interpolated normal is exactly zero with weights fp32 holds exactly (elsewhere a
  # cancellation leaves a few ulps in fp32, whose direction is arbitrary; the bound above is infinite there)
  nv = n[f[owner]].astype(np.float64)
  zero = ~(w[:, :, None] * nv).sum(1).any(1) & ((w == 0.5) | (w == 1) | ~nv.any(2)).all(1)
  e1 = v[f[owner, 1]].astype(np.float64) - v[f[owner, 0]]
  e2 = v[f[owner, 2]].astype(np.float64) - v[f[owner, 0]]
  flat = ~np.cross(e1, e2).any(1)
  assert (zero & ~flat).sum() > 20 and (zero & flat).sum() > 20
  assert np.array_equal(normals[zero & flat], np.tile(np.float32([0, 0, 1]), ((zero & flat).sum(), 1)))
  g = np.cross(e1, e2)[zero & ~flat]
  g /= np.linalg.norm(g, axis=1, keepdims=True)
  assert np.abs(normals[zero & ~flat] - g).max() < 1e-5
  # corner texels: their vertices, bit for bit
  pos = np.full(size * size, -1, np.int64)
  pos[index] = np.arange(len(index))
  t = pos[np.floor(uv[..., 1]).astype(np.int64) * size + np.floor(uv[..., 0]).astype(np.int64)]
  assert (t >= 0).all() and np.array_equal(points[t].view(np.uint32), v[f].view(np.uint32))
  # the ownership invariant on the kernel's outputs: bilinear samples inside each face read its texels only
  owner_map = np.full(size * size, -1, np.int64)
  owner_map[index] = owner
  rng = np.random.default_rng(c)
  faces = rng.integers(0, len(f), 100000)
  bary = rng.dirichlet((1, 1, 1), len(faces))
  p = (bary[:, :, None] * uv[faces].astype(np.float64)).sum(1)
  xs, ys = R.bilinear_texels(p[:, 0], p[:, 1])
  got = owner_map[np.where(xs >= 0, ys * size + xs, 0)]
  assert (np.where(xs >= 0, got, faces[:, None]) == faces[:, None]).all()


def test_raster_rejects_bad_arguments(mods):
  lib, ops, _ = mods
  v, f, n = (torch.tensor(a, device='cuda') for a in _special_mesh(F=8))
  with pytest.raises(ValueError, match='texture size'):
    ops.mesh_texture_raster(v, f, n, 3)
  with pytest.raises(ValueError, match=r'9 faces .*at most 8 faces'):
    ops.mesh_texture_raster(v, torch.cat([f, f[:1]]), n, 8)
  bad = f.clone()
  bad[3, 1] = v.shape[0]
  with pytest.raises(ValueError, match='face index'):
    ops.mesh_texture_raster(v, bad, n, 64)
  bad[3, 1] = -1
  with pytest.raises(ValueError, match='face index'):
    ops.mesh_texture_raster(v, bad, n, 64)
  with pytest.raises(ValueError, match='normals'):
    ops.mesh_texture_raster(v, f, n[:-1], 64)
  uv, index, points, normals = ops.mesh_texture_raster(v, f[:0], n, 64)
  assert uv.shape == (0, 3, 2) and index.shape == (0,) and points.shape == (0, 3)
  L = lib.load()
  P = lib.ptr
  s = lib.stream_ptr()
  out = [torch.empty(8 * 3 * 2, device='cuda'), torch.empty(4 * 256, dtype=torch.int32, device='cuda'),
         torch.empty(4 * 256, 3, device='cuda'), torch.empty(4 * 256, 3, device='cuda')]
  call = lambda nv=v.shape[0], nf=8, vert=v, size=64, o=out: L.mnrf_mesh_texture_raster(
      nv, nf, P(vert), P(f), P(n), size, *(P(t) for t in o), s)
  assert call() == 0 and call(nf=0) == 0
  for kw in (dict(nv=-1), dict(nf=-1), dict(size=3), dict(size=16385), dict(size=7, nf=3), dict(vert=None),
             dict(nv=0), dict(o=out[:3] + [None]), dict(o=[None] + out[1:])):
    assert call(**kw) != 0, kw
  torch.cuda.synchronize()


def _stripes(points):
  """An analytic colour with stripes about 4 grid units apart: uint8 [N, 3] and its Lipschitz constant per unit
  length in [0, 1] colour units."""
  k = 1.6
  p = points.double()
  rgb = torch.stack([0.5 + 0.5 * torch.sin(k * (p[:, 0] + p[:, 1])), 0.5 + 0.5 * torch.sin(k * (p[:, 1] - p[:, 2])),
                     0.5 + 0.5 * torch.cos(k * p[:, 2])], -1)
  return rgb, 0.5 * k * np.sqrt(2)


def test_texture_beats_vertex_colours(mods):
  """A marching-cubes sphere simplified to about 20 k faces, coloured by an analytic field: the bilinear texture
  sample at random points of random faces stays within the field's Lipschitz constant times the texel's reach in
  space plus 1/255, and its mean error is well below that of the vertex colours interpolated barycentrically."""
  _, ops, mesh = mods
  grid = torch.tensor(sphere((128, 128, 128), (63.6, 64.2, 63.3), 50.3), device='cuda')
  v, f, n = ops.marching_cubes(grid, 0.0, normals=True)
  v, f, n = mesh.simplify_mesh(v, f, n, target_faces=20000)
  assert 19000 <= len(f) <= 20001
  size = 11 * ops.texture_atlas(len(f), 4096)[0]
  color_fn = lambda p, nn: (_stripes(p)[0] * 255).round().to(torch.uint8)
  uv, tex = mesh.bake_texture(v, f, n, size, color_fn)
  assert ops.texture_atlas(len(f), size)[1] == 11
  rng = np.random.default_rng(0)
  N = 200000
  faces = rng.integers(0, len(f), N)
  bary = rng.dirichlet((1, 1, 1), N)
  vh, fh, uvh = (t.cpu().numpy().astype(np.float64) for t in (v, f, uv))
  fh = fh.astype(np.int64)
  pts = (bary[:, :, None] * vh[fh[faces]]).sum(1)
  q = (bary[:, :, None] * uvh[faces]).sum(1)
  want, lip = _stripes(torch.tensor(pts))
  want = want.numpy()
  got = R.bilinear_sample(tex.cpu().numpy(), q[:, 0], q[:, 1]) / 255
  # reach: a texel read lies within sqrt(2) texels of the sample in UV; its point is the chart's nearest point, no
  # farther; one texel of UV spans at most the largest singular value of the face's UV-to-space map
  d = np.abs(uvh[:, 1, 0] - uvh[:, 0, 0])
  J = np.stack([vh[fh[:, 1]] - vh[fh[:, 0]], vh[fh[:, 2]] - vh[fh[:, 0]]], -1) / d[:, None, None]
  smax = np.linalg.svd(J, compute_uv=False)[:, 0]
  err = np.abs(got - want).max(1)
  assert (err <= lip * np.sqrt(2) * smax[faces] + 1 / 255 + 1e-9).all()
  vcol = (_stripes(v)[0] * 255).round().cpu().numpy() / 255
  verr = np.abs((bary[:, :, None] * vcol[fh[faces]]).sum(1) - want).max(1)
  assert err.mean() < 0.25 * verr.mean(), (err.mean(), verr.mean())


def _corner_check(v, f, n, uv, tex, want_rgb, size):
  """Each corner texel: its raster point is its vertex bit for bit, its colour within one code of want_rgb."""
  from multinerf_b200 import ops
  uv2, index, points, _ = ops.mesh_texture_raster(v, f, n, size)
  assert torch.equal(uv2, uv)
  pos = torch.full((size * size,), -1, dtype=torch.int64, device='cuda')
  pos[index.long()] = torch.arange(len(index), device='cuda')
  cell = uv.floor().long()
  flat = cell[..., 1] * size + cell[..., 0]
  t = pos[flat]
  assert (t >= 0).all()
  assert torch.equal(points[t].view(torch.int32), v[f.long()].view(torch.int32))
  got = tex.view(-1, 3)[flat].int()
  assert (got - want_rgb[f.long()].int()).abs().max() <= 1


def _equal(a, b):
  assert len(a) == len(b)
  for x, y in zip(a, b):
    assert x.dtype == y.dtype and torch.equal(x, y)


def test_extract_mesh_with_texture(mods, scene):
  _, _, mesh = mods
  model, _ = scene
  bbox, res = (-1.5, -1.5, -1.5, 1.5, 1.5, 1.5), 48
  grid, h = mesh.density_grid(model, bbox, res)
  level = float(grid.median())
  for colors in (False, True):
    for target in (0, 3000):
      kw = dict(colors=colors, keep_components=2, target_faces=target)
      base = mesh.extract_mesh(model, bbox, res, level, **kw)
      seen = []
      got = mesh.extract_mesh(model, bbox, res, level, texture_size=4096, before_texture=lambda *a: seen.append(a),
                              **kw)
      assert len(got) == 6 and len(seen) == 1 and all(x is y for x, y in zip(seen[0], got[:4]))
      _equal(got[:2], base[:2])
      normals = mesh.extract_mesh(model, bbox, res, level, colors=True, keep_components=2, target_faces=target)[2]
      assert torch.equal(got[2], normals)
      if colors:
        _equal(got[2:4], base[2:4])
      else:
        assert got[3] is None
      v, f, n, _, uv, tex = got
      assert tex.shape == (4096, 4096, 3) and tex.dtype == torch.uint8
      _corner_check(v, f, n, uv, tex, mesh.vertex_colors(model, v, n, h * h / 12), 4096)
  with pytest.raises(ValueError, match='at most 8 faces.*mesh_target_faces'):
    mesh.extract_mesh(model, bbox, res, level, texture_size=8)


def test_extract_mesh_tsdf_with_texture(mods, scene):
  _, _, mesh = mods
  model, dataset = scene
  bbox, res = (-1.5, -1.5, -1.5, 1.5, 1.5, 1.5), 40
  state, h = mesh.fuse_tsdf(mesh.render_views(model, dataset), dataset.cameras, dataset.camtype, bbox, res, 3.0,
                            colors=True, device=model.device)
  lo = torch.tensor(bbox[:3], device='cuda')
  for colors in (False, True):
    for target in (0, 2000):
      kw = dict(colors=colors, keep_components=1, target_faces=target)
      base = mesh.extract_mesh_tsdf(model, dataset, bbox, res, **kw)
      got = mesh.extract_mesh_tsdf(model, dataset, bbox, res, texture_size=2048, **kw)
      assert len(got) == 6
      _equal(got[:2], base[:2])
      assert torch.equal(got[2], mesh.tsdf_mesh(state, bbox, h, colors=True, clean_args=dict(keep_components=1),
                                                target_faces=target)[2])
      if colors:
        _equal(got[2:4], base[2:4])
      v, f, n, _, uv, tex = got
      _corner_check(v, f, n, uv, tex, mesh.tsdf_colors(state[2], state[3], (v - lo) / h), 2048)
      assert len(torch.unique(tex.view(-1, 3), dim=0)) > 2


def test_extract_mesh_script_writes_textured_obj(tmp_path, capsys):
  """extract_mesh.py with mesh_texture_size after a short train.py run: the PLY byte for byte as without it, then
  the OBJ, MTL and PNG with the counts the texture line prints."""
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  sys.path.insert(0, root)
  from PIL import Image
  from multinerf_b200 import lib
  lib.require_device()
  import extract_mesh as mesh_script
  import train as train_script
  from test_gpu_mesh import _write_scene
  from test_mesh_texture_cpu import read_obj
  data, ckpt = str(tmp_path / 'scene'), str(tmp_path / 'ckpt')
  _write_scene(data)
  steps = 40
  bindings = [f"Config.data_dir = '{data}'", f"Config.checkpoint_dir = '{ckpt}'", 'Config.batch_size = 1024',
              f'Config.max_steps = {steps}', 'Config.print_every = 20', f'Config.checkpoint_every = {steps}',
              f'Config.train_render_every = {10 * steps}', 'Config.render_chunk_size = 512', 'Config.near = 1.5',
              'Config.far = 5.0', "Config.dataset_loader = 'blender'", 'Model.num_prop_samples = 32',
              'Model.num_nerf_samples = 16', 'PropMLP.net_depth = 2', 'PropMLP.net_width = 64',
              'NerfMLP.net_depth = 4', 'NerfMLP.net_width = 128', 'NerfMLP.bottleneck_width = 64',
              'NerfMLP.net_width_viewdirs = 64', 'PropMLP.disable_density_normals = True',
              'PropMLP.disable_rgb = True', 'NerfMLP.disable_density_normals = True']
  argv = [f'--gin_bindings={b}' for b in bindings]
  train_script.main(argv)
  capsys.readouterr()
  mesh_argv = argv + ['--gin_bindings=Config.mesh_resolution = 40', '--gin_bindings=Config.mesh_level = 0.5',
                      '--gin_bindings=Config.mesh_target_faces = 2000']
  path = mesh_script.main(mesh_argv)
  plain = open(path, 'rb').read()
  plain_lines = capsys.readouterr().out.splitlines()
  os.remove(path)
  assert mesh_script.main(mesh_argv + ['--gin_bindings=Config.mesh_texture_size = 512']) == path
  lines = capsys.readouterr().out.splitlines()
  assert open(path, 'rb').read() == plain
  assert [l.split(' in ')[0] for l in lines[:-1]] == [l.split(' in ')[0] for l in plain_lines]
  tex_line = lines[-1]
  stem = os.path.splitext(path)[0]
  assert tex_line.startswith('texture 512 x 512, ') and tex_line.endswith(f'-> {stem}.obj'), tex_line
  c = int(tex_line.split(', ')[1].split(' x ')[0])
  T = int(tex_line.split('texels per cell, ')[1].split(' texels')[0])
  v, vt, vn, f, mtllib, _ = read_obj(stem + '.obj')
  assert mtllib == os.path.basename(stem) + '.mtl' and os.path.exists(stem + '.mtl')
  assert len(vt) == 3 * len(f) and len(vn) == len(v) and T == (len(f) + 1) // 2 * c * c and c >= 4
  img = np.asarray(Image.open(stem + '.png'))
  assert img.shape == (512, 512, 3) and len(np.unique(img.reshape(-1, 3), axis=0)) > 2
  with pytest.raises(ValueError, match='mesh_target_faces'):
    mesh_script.main(mesh_argv + ['--gin_bindings=Config.mesh_texture_size = 16'])
  assert open(path, 'rb').read() == plain
