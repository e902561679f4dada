"""Parameter surface of the hot path: `Config`, `Model`/`NerfMLP`/`PropMLP` fields, gin subset.

Mirrors the reference's configurable names and defaults so that the shipped
`configs/*.gin` files bind unmodified:
  Config   internal/configs.py:45-172      Model  internal/models.py:50-72
  MLP      internal/models.py:343-379      loader internal/configs.py:183-192
gin-config is not installed in this image; `parse_gin` implements exactly the syntax
the reference's config files use: `Class.attr = literal`, `@module.fn` references
(kept as the function's short name, e.g. '@jnp.reciprocal' -> 'reciprocal'),
`#` comments and `include 'file.gin'`; unknown classes/attrs are skipped
(`skip_unknown=True`, configs.py:186).
"""
import ast
import dataclasses
import os
from typing import Any, Dict, Optional, Tuple


@dataclasses.dataclass
class Config:
  """Fields of internal/configs.py:45-172 that reach the hot path or its closure."""
  dataset_loader: str = 'llff'
  batching: str = 'all_images'
  batch_size: int = 16384
  patch_size: int = 1
  factor: int = 0
  compute_disp_metrics: bool = False
  compute_normal_metrics: bool = False
  disable_multiscale_loss: bool = False
  randomized: bool = True
  near: float = 2.
  far: float = 6.
  checkpoint_dir: Optional[str] = None
  render_dir: Optional[str] = None
  data_dir: Optional[str] = None
  render_chunk_size: int = 16384
  vis_num_rays: int = 16
  max_steps: int = 250000
  early_exit_steps: Optional[int] = None
  checkpoint_every: int = 25000
  print_every: int = 100
  train_render_every: int = 5000
  cast_rays_in_train_step: bool = False
  # rays per forward/backward pass of a train step, per process (0: the whole per-process batch in one pass); the
  # passes accumulate into one gradient, so a batch larger than device memory trains at its configured size
  train_chunk_size: int = 0
  data_loss_type: str = 'charb'
  charb_padding: float = 0.001
  data_loss_mult: float = 1.0
  data_coarse_loss_mult: float = 0.
  interlevel_loss_mult: float = 1.0
  orientation_loss_mult: float = 0.0
  orientation_coarse_loss_mult: float = 0.0
  orientation_loss_target: str = 'normals_pred'
  predicted_normal_loss_mult: float = 0.0
  predicted_normal_coarse_loss_mult: float = 0.0
  weight_decay_mults: Dict[str, Any] = dataclasses.field(default_factory=dict)
  lr_init: float = 0.002
  lr_final: float = 0.00002
  lr_delay_steps: int = 512
  lr_delay_mult: float = 0.01
  adam_beta1: float = 0.9
  adam_beta2: float = 0.999
  adam_eps: float = 1e-6
  grad_max_norm: float = 0.001
  grad_max_val: float = 0.
  distortion_loss_mult: float = 0.01
  rawnerf_mode: bool = False
  apply_bayer_mask: bool = False
  forward_facing: bool = False
  eval_render_interval: int = 1
  # --- fields used by the callers either side of the hot path (datasets / train / eval / render;
  #     internal/configs.py:54-172), same names and defaults
  load_alphabetical: bool = True
  render_path: bool = False
  llffhold: int = 8
  llff_use_all_images_for_training: bool = False
  use_tiffs: bool = False
  gc_every: int = 10000
  vocab_tree_path: Optional[str] = None
  num_showcase_images: int = 5
  deterministic_showcase: bool = True
  vis_decimate: int = 0
  robustnerf_inlier_quantile: float = 0.5
  enable_robustnerf_loss: bool = False
  robustnerf_inner_patch_size: int = 8
  robustnerf_smoothed_filter_size: int = 3
  robustnerf_smoothed_inlier_quantile: float = 0.5
  robustnerf_inner_patch_inlier_quantile: float = 0.5
  eval_only_once: bool = True
  eval_save_output: bool = True
  eval_save_ray_data: bool = False
  eval_dataset_limit: int = 2 ** 31 - 1
  eval_quantize_metrics: bool = True
  eval_crop_borders: int = 0
  render_video_fps: int = 60
  render_video_crf: int = 18
  render_path_frames: int = 120
  z_variation: float = 0.
  z_phase: float = 0.
  render_dist_percentile: float = 0.5
  render_dist_curve_fn: str = 'log'
  render_path_file: Optional[str] = None
  render_job_id: int = 0
  render_num_jobs: int = 1
  render_resolution: Optional[Tuple[int, int]] = None
  render_focal: Optional[float] = None
  render_camtype: Optional[str] = None
  render_spherical: bool = False
  render_save_async: bool = True
  render_spline_keyframes: Optional[str] = None
  render_spline_n_interp: int = 30
  render_spline_degree: int = 5
  render_spline_smoothness: float = .03
  render_spline_interpolate_exposure: bool = False
  exposure_percentile: float = 97.
  num_border_pixels_to_mask: int = 0
  autoexpose_renders: bool = False
  eval_raw_affine_cc: bool = False
  # extract_mesh.py (multinerf_b200/mesh.py): grid points along the longest side of the box (cells are cubes), the
  # density level of the surface, and the box (x0, y0, z0, x1, y1, z1) in world coordinates; None: [-1.5, 1.5]^3,
  # or [-1, 1]^3 under the scene contraction.  Forward-facing (NDC) scenes need an explicit box.
  mesh_resolution: int = 512
  mesh_level: float = 10.
  mesh_bbox: Optional[Tuple[float, ...]] = None
  # also write vertex normals and colours (each vertex's radiance seen head-on from outside, GLO zeroed)
  mesh_vertex_colors: bool = False
  # 'density': marching cubes on the density grid at mesh_level; 'tsdf': render the training views, fuse their
  # median distances into a truncated signed-distance grid and mesh its zero crossing (no level to choose; vertex
  # colours are the rendered colours).  mesh_tsdf_truncation: the band, in cells (>= 1).
  mesh_method: str = 'density'
  mesh_tsdf_truncation: float = 3.
  # cleaning, right after marching cubes (mesh.clean_mesh); 0 turns each off.  mesh_min_views: drop vertices that
  # land on the images of fewer training views (frustum culling, no occlusion; not NDC) and the faces using them.
  # mesh_keep_components: then keep only this many connected components, the largest by face count.
  mesh_min_views: int = 0
  mesh_keep_components: int = 0
  # simplification, right after cleaning (mesh.simplify_mesh): quadric edge collapse down to about this many faces;
  # 0 turns it off.
  mesh_target_faces: int = 0
  # texture, after simplification (mesh.bake_texture): the side in texels, in [4, 16384], of a texture atlas the
  # surface colour is baked into, written beside the PLY as mesh_step_<step>.{obj,mtl,png}; 0 turns it off.
  mesh_texture_size: int = 0
  # score the extracted mesh against the test views (mesh.evaluate_mesh): trace every test pixel's ray into it, write
  # its colour, normal and distance renders and per-image metrics (psnr / ssim against the test images, and
  # coverage, spurious hits and depth error against the NeRF's own renders) to <checkpoint_dir>/mesh/eval_step_<step>.
  # Not for forward-facing (NDC) scenes.
  mesh_eval: bool = False
  # the space of the extraction grid: 'world', or 'contracted' for unbounded scenes under the scene contraction
  # (coord.contract; not NDC): the grid then lies in contracted coordinates, so the background is meshed too.  There,
  # mesh_bbox is read in contracted coordinates (None: [-2, 2]^3, all of contracted space; a grid of
  # mesh_resolution points over it has half the foreground resolution of the world default), mesh_level is a
  # density per unit of contracted length (the same inside the unit ball), and the TSDF band is in contracted cells.
  # Meshes are written in world coordinates either way.
  mesh_space: str = 'world'


@dataclasses.dataclass
class ModelConfig:
  """internal/models.py:50-72 (gin name `Model`)."""
  num_prop_samples: int = 64
  num_nerf_samples: int = 32
  num_levels: int = 3
  bg_intensity_range: Tuple[float, float] = (1., 1.)
  anneal_slope: float = 10
  stop_level_grad: bool = True
  use_viewdirs: bool = True
  raydist_fn: Optional[str] = None        # None | 'piecewise' | reciprocal/log/exp/sqrt/square
  ray_shape: str = 'cone'
  disable_integration: bool = False
  single_jitter: bool = True
  dilation_multiplier: float = 0.5
  dilation_bias: float = 0.0025
  num_glo_features: int = 0
  num_glo_embeddings: int = 1000
  learned_exposure_scaling: bool = False
  near_anneal_rate: Optional[float] = None
  near_anneal_init: float = 0.95
  single_mlp: bool = False
  resample_padding: float = 0.0
  use_gpu_resampling: bool = False
  opaque_background: bool = False


@dataclasses.dataclass
class MLPConfig:
  """internal/models.py:343-379 (gin names `NerfMLP` / `PropMLP`)."""
  net_depth: int = 8
  net_width: int = 256
  bottleneck_width: int = 256
  net_depth_viewdirs: int = 1
  net_width_viewdirs: int = 128
  net_activation: str = 'relu'
  min_deg_point: int = 0
  max_deg_point: int = 12
  weight_init: str = 'he_uniform'
  skip_layer: int = 4
  skip_layer_dir: int = 4
  num_rgb_channels: int = 3
  deg_view: int = 4
  use_reflections: bool = False
  use_directional_enc: bool = False
  enable_pred_roughness: bool = False
  roughness_activation: str = 'softplus'
  roughness_bias: float = -1.
  use_diffuse_color: bool = False
  use_specular_tint: bool = False
  use_n_dot_v: bool = False
  bottleneck_noise: float = 0.0
  density_activation: str = 'softplus'
  density_bias: float = -1.
  density_noise: float = 0.
  rgb_premultiplier: float = 1.
  rgb_activation: str = 'sigmoid'
  rgb_bias: float = 0.
  rgb_padding: float = 0.001
  enable_pred_normals: bool = False
  disable_density_normals: bool = False
  disable_rgb: bool = False
  warp_fn: Optional[str] = None           # None | 'contract'
  basis_shape: str = 'icosahedron'
  basis_subdivisions: int = 2

  def validate(self):
    # internal/models.py:383-385
    if self.use_reflections and not (self.enable_pred_normals or
                                     not self.disable_density_normals):
      raise ValueError('Normals must be computed for reflection directions.')


@dataclasses.dataclass
class Bundle:
  """Everything gin would have bound: Config + Model + NerfMLP + PropMLP."""
  config: Config = dataclasses.field(default_factory=Config)
  model: ModelConfig = dataclasses.field(default_factory=ModelConfig)
  nerf_mlp: MLPConfig = dataclasses.field(default_factory=MLPConfig)
  prop_mlp: MLPConfig = dataclasses.field(default_factory=MLPConfig)


_GIN_CLASSES = {'Config': 'config', 'Model': 'model', 'NerfMLP': 'nerf_mlp',
                'PropMLP': 'prop_mlp'}


def _parse_value(text):
  text = text.strip()
  if text.startswith('@'):
    name = text[1:].rstrip('()').strip()
    return name.split('.')[-1]
  try:
    return ast.literal_eval(text)
  except (ValueError, SyntaxError) as e:
    raise ValueError(f'gin subset: cannot parse value {text!r}') from e


def _strip_comment(line):
  out, quote = [], None
  for ch in line:
    if quote:
      if ch == quote:
        quote = None
    elif ch in '\'"':
      quote = ch
    elif ch == '#':
      break
    out.append(ch)
  return ''.join(out).strip()


def parse_gin(text, bundle=None, search_paths=(), skip_unknown=True):
  """Apply gin-subset `text` onto `bundle` (a fresh Bundle when None)."""
  bundle = bundle or Bundle()
  pending = ''
  for raw in text.splitlines():
    line = _strip_comment(raw)
    if not line:
      continue
    line = pending + line
    if line.count('(') > line.count(')') or line.count('[') > line.count(']') or \
       line.count('{') > line.count('}'):
      pending = line + ' '
      continue
    pending = ''
    if line.startswith('include '):
      fname = ast.literal_eval(line[len('include '):].strip())
      for base in list(search_paths) + ['.']:
        cand = os.path.join(base, fname)
        if not os.path.exists(cand):
          cand = os.path.join(base, os.path.basename(fname))
        if os.path.exists(cand):
          with open(cand) as f:
            parse_gin(f.read(), bundle, search_paths, skip_unknown)
          break
      else:
        raise FileNotFoundError(f'gin include {fname!r} not found in {search_paths}')
      continue
    if '=' not in line:
      raise ValueError(f'gin subset: not a binding: {raw!r}')
    lhs, rhs = line.split('=', 1)
    lhs = lhs.strip()
    if '/' in lhs:                       # scope prefix (train/eval): bind regardless
      lhs = lhs.split('/')[-1]
    if '.' not in lhs:
      raise ValueError(f'gin subset: macro bindings are not supported: {raw!r}')
    cls, attr = lhs.rsplit('.', 1)
    target = _GIN_CLASSES.get(cls.split('.')[-1])
    if target is None or not hasattr(getattr(bundle, target), attr):
      if skip_unknown:
        continue
      raise ValueError(f'gin subset: unknown configurable {lhs!r}')
    setattr(getattr(bundle, target), attr, _parse_value(rhs))
  return bundle


def load_config(gin_configs=(), gin_bindings=(), search_paths=()):
  """Counterpart of internal/configs.py:183-192: files first, then bindings."""
  bundle = Bundle()
  for path in gin_configs or ():
    with open(path) as f:
      parse_gin(f.read(), bundle, list(search_paths) + [os.path.dirname(path)])
  for b in gin_bindings or ():
    parse_gin(b, bundle, search_paths)
  bundle.nerf_mlp.validate()
  bundle.prop_mlp.validate()
  return bundle


# The four BASELINE configs, written as gin text with the same bindings as the
# reference's configs/{360,blender_256,blender_refnerf,llff_raw}.gin so they are usable
# on a box where /root/reference does not exist.
GIN_360 = """
Config.dataset_loader = 'llff'
Config.near = 0.2
Config.far = 1e6
Config.factor = 4
Model.raydist_fn = @jnp.reciprocal
Model.opaque_background = True
PropMLP.warp_fn = @coord.contract
PropMLP.net_depth = 4
PropMLP.net_width = 256
PropMLP.disable_density_normals = True
PropMLP.disable_rgb = True
NerfMLP.warp_fn = @coord.contract
NerfMLP.net_depth = 8
NerfMLP.net_width = 1024
NerfMLP.disable_density_normals = True
"""

GIN_BLENDER_256 = """
Config.dataset_loader = 'blender'
Config.batching = 'single_image'
Config.near = 2
Config.far = 6
Config.eval_render_interval = 5
Config.data_loss_type = 'mse'
Config.adam_eps = 1e-8
Model.num_levels = 2
Model.num_prop_samples = 128
Model.num_nerf_samples = 32
PropMLP.net_depth = 4
PropMLP.net_width = 256
PropMLP.basis_shape = 'octahedron'
PropMLP.basis_subdivisions = 1
PropMLP.disable_density_normals = True
PropMLP.disable_rgb = True
NerfMLP.net_depth = 8
NerfMLP.net_width = 256
NerfMLP.basis_shape = 'octahedron'
NerfMLP.basis_subdivisions = 1
NerfMLP.disable_density_normals = True
Config.distortion_loss_mult = 0.
NerfMLP.max_deg_point = 16
PropMLP.max_deg_point = 16
"""


GIN_LLFF_RAW = """
Config.dataset_loader = 'llff'
Config.near = 0.
Config.far = 1.
Config.factor = 4
Config.forward_facing = True
Model.ray_shape = 'cylinder'
PropMLP.net_depth = 4
PropMLP.net_width = 256
PropMLP.basis_shape = 'octahedron'
PropMLP.basis_subdivisions = 1
PropMLP.disable_density_normals = True
PropMLP.disable_rgb = True
NerfMLP.net_depth = 8
NerfMLP.net_width = 256
NerfMLP.basis_shape = 'octahedron'
NerfMLP.basis_subdivisions = 1
NerfMLP.disable_density_normals = True
NerfMLP.max_deg_point = 16
PropMLP.max_deg_point = 16
Config.rawnerf_mode = True
Config.data_loss_type = 'rawnerf'
Config.apply_bayer_mask = True
Model.learned_exposure_scaling = True
Model.num_levels = 2
Model.num_prop_samples = 128
Model.num_nerf_samples = 128
Model.opaque_background = True
NerfMLP.rgb_padding = 0.
NerfMLP.rgb_activation = @math.safe_exp
NerfMLP.rgb_bias = -5.
PropMLP.rgb_padding = 0.
PropMLP.rgb_activation = @math.safe_exp
PropMLP.rgb_bias = -5.
Config.interlevel_loss_mult = .0
Config.distortion_loss_mult = .01
Config.orientation_loss_mult = 0.
Config.data_coarse_loss_mult = 0.1
NerfMLP.density_noise = 1.
PropMLP.density_noise = 1.
Model.single_mlp = True
Model.anneal_slope = 0.
Model.dilation_multiplier = 0.
Model.dilation_bias = 0.
Model.single_jitter = False
NerfMLP.weight_init = 'glorot_uniform'
PropMLP.weight_init = 'glorot_uniform'
Config.batch_size = 16384
Config.render_chunk_size = 16384
Config.lr_init = 1e-3
Config.lr_final = 1e-5
Config.max_steps = 500000
Config.checkpoint_every = 25000
Config.lr_delay_steps = 2500
Config.lr_delay_mult = 0.01
Config.grad_max_norm = 0.1
Config.grad_max_val = 0.1
Config.adam_eps = 1e-8
"""


GIN_BLENDER_REFNERF = """
Config.dataset_loader = 'blender'
Config.batching = 'single_image'
Config.near = 2
Config.far = 6
Config.eval_render_interval = 5
Config.compute_normal_metrics = True
Config.data_loss_type = 'mse'
Config.distortion_loss_mult = 0.0
Config.orientation_loss_mult = 0.1
Config.orientation_loss_target = 'normals_pred'
Config.predicted_normal_loss_mult = 3e-4
Config.orientation_coarse_loss_mult = 0.01
Config.predicted_normal_coarse_loss_mult = 3e-5
Config.interlevel_loss_mult = 0.0
Config.data_coarse_loss_mult = 0.1
Config.adam_eps = 1e-8
Model.num_levels = 2
Model.single_mlp = True
Model.num_prop_samples = 128
Model.num_nerf_samples = 128
Model.anneal_slope = 0.
Model.dilation_multiplier = 0.
Model.dilation_bias = 0.
Model.single_jitter = False
Model.resample_padding = 0.01
NerfMLP.net_depth = 8
NerfMLP.net_width = 256
NerfMLP.net_depth_viewdirs = 8
NerfMLP.basis_shape = 'octahedron'
NerfMLP.basis_subdivisions = 1
NerfMLP.disable_density_normals = False
NerfMLP.enable_pred_normals = True
NerfMLP.use_directional_enc = True
NerfMLP.use_reflections = True
NerfMLP.deg_view = 5
NerfMLP.enable_pred_roughness = True
NerfMLP.use_diffuse_color = True
NerfMLP.use_specular_tint = True
NerfMLP.use_n_dot_v = True
NerfMLP.bottleneck_width = 128
NerfMLP.density_bias = 0.5
NerfMLP.max_deg_point = 16
"""


def bundle_blender_refnerf():
  return parse_gin(GIN_BLENDER_REFNERF)


def bundle_llff_raw():
  return parse_gin(GIN_LLFF_RAW)


def bundle_360():
  return parse_gin(GIN_360)


def bundle_blender_256():
  return parse_gin(GIN_BLENDER_256)
