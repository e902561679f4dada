"""Dataset loaders feeding the hot path (reference: internal/datasets.py).

Same public surface: `load_dataset(split, data_dir, config)` -> an iterator that yields
`utils.Batch` objects -- random-ray training batches (`split='train'`) or one full test image per
`next()` (`split='test'`) -- with the attributes train.py / eval.py / render.py read (`size`,
`cameras`, `camtype`, `metadata`, `height`, `width`, `near`, `far`, ...).

Differences from the reference's host pipeline:
  * the reference's loader thread also casts the rays with numpy (datasets.py:452-455); here the thread only
    draws PIXELS (coordinates, camera indices, colours) and `__next__` turns them into rays with ONE
    launch of `mnrf_pixels_to_rays` on the device (or hands the pixels to the train step when
    `cast_rays_in_train_step` is set) -- there is no CPU ray-casting path; a panorama
    (`render_camtype='pano'`) is queued as its camera index and cast by `mnrf_spherical_rays`;
  * one process per GPU: every process draws `batch_size // world_size` rays from its own numpy
    stream (the reference seeds `20201473 + host_id`, train.py:47), nothing is re-sharded afterwards.

COLMAP sparse models (`sparse/0/{cameras,images}.bin`) are parsed by a small reader of the published
binary layout (the reference vendors `pycolmap` for this, datasets.py:36-39).
"""
import abc
import copy
import json
import os
import queue
import struct
import threading

import numpy as np
import torch

from . import camera_utils
from . import image as lib_image
from . import utils


def load_dataset(split, train_dir, config, device=None, rank=0, world=1):
  """datasets.py:42-51."""
  table = {'blender': Blender, 'llff': LLFF, 'tat_nerfpp': TanksAndTemplesNerfPP,
           'tat_fvs': TanksAndTemplesFVS, 'dtu': DTU}
  if config.dataset_loader not in table:
    raise KeyError(f'unknown dataset_loader {config.dataset_loader!r}')
  return table[config.dataset_loader](split, train_dir, config, device=device, rank=rank, world=world)


# ------------------------------------------------------------------------------------------ COLMAP
_COLMAP_MODELS = {0: ('SIMPLE_PINHOLE', 3), 1: ('PINHOLE', 4), 2: ('SIMPLE_RADIAL', 4), 3: ('RADIAL', 5),
                  4: ('OPENCV', 8), 5: ('OPENCV_FISHEYE', 8), 6: ('FULL_OPENCV', 12), 7: ('FOV', 5),
                  8: ('SIMPLE_RADIAL_FISHEYE', 4), 9: ('RADIAL_FISHEYE', 5), 10: ('THIN_PRISM_FISHEYE', 12)}


def _qvec_to_rot(q):
  w, x, y, z = q
  return np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                   [2 * x * y + 2 * w * z, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * w * x],
                   [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x * x - 2 * y * y]])


def read_colmap_model(sparse_dir):
  """Cameras and images of a COLMAP binary sparse model.
  Returns (cameras {id: (model_name, width, height, params)}, images [(name, qvec, tvec, camera_id)] in
  file order)."""
  cams = {}
  with open(os.path.join(sparse_dir, 'cameras.bin'), 'rb') as f:
    (n,) = struct.unpack('<Q', f.read(8))
    for _ in range(n):
      cam_id, model_id, w, h = struct.unpack('<iiQQ', f.read(24))
      name, npar = _COLMAP_MODELS[model_id]
      cams[cam_id] = (name, w, h, struct.unpack('<' + 'd' * npar, f.read(8 * npar)))
  images = []
  with open(os.path.join(sparse_dir, 'images.bin'), 'rb') as f:
    (n,) = struct.unpack('<Q', f.read(8))
    for _ in range(n):
      vals = struct.unpack('<idddddddi', f.read(64))
      name = b''
      while True:
        c = f.read(1)
        if c == b'\x00':
          break
        name += c
      (n2d,) = struct.unpack('<Q', f.read(8))
      f.seek(24 * n2d, 1)                                # (x, y, point3D_id) triples
      images.append((name.decode('utf-8'), np.array(vals[1:5]), np.array(vals[5:8]), vals[8]))
  return cams, images


def load_colmap_posedata(colmap_dir):
  """NeRF-style pose data from a COLMAP model (datasets.py:54-149 `NeRFSceneManager.process`): shared
  intrinsics of camera 1, camera-to-world matrices in the (right, up, back) convention, distortion
  parameters by camera model.  Returns (names, poses [N,3,4], pixtocam [3,3], params, camtype)."""
  cams, images = read_colmap_model(colmap_dir)
  model, _, _, prm = cams[1]
  if model in ('SIMPLE_PINHOLE', 'SIMPLE_RADIAL', 'RADIAL'):
    fx = fy = prm[0]
    cx, cy = prm[1], prm[2]
    rest = prm[3:]
  else:
    fx, fy, cx, cy = prm[:4]
    rest = prm[4:]
  pixtocam = np.linalg.inv(camera_utils.intrinsic_matrix(fx, fy, cx, cy))
  w2c = []
  for _, q, t, _ in images:
    m = np.eye(4)
    m[:3, :3] = _qvec_to_rot(q)
    m[:3, 3] = t
    w2c.append(m)
  poses = np.linalg.inv(np.stack(w2c))[:, :3, :4]
  names = [im[0] for im in images]
  poses = poses @ np.diag([1, -1, -1, 1])                # COLMAP (right, down, fwd) -> NeRF (right, up, back)
  params, camtype = None, camera_utils.ProjectionType.PERSPECTIVE
  zero = lambda keys: {k: 0. for k in keys}
  if model == 'SIMPLE_RADIAL':
    params = zero(['k1', 'k2', 'k3', 'p1', 'p2'])
    params['k1'] = rest[0]
  elif model == 'RADIAL':
    params = zero(['k1', 'k2', 'k3', 'p1', 'p2'])
    params['k1'], params['k2'] = rest[0], rest[1]
  elif model == 'OPENCV':
    params = zero(['k1', 'k2', 'k3', 'p1', 'p2'])
    params['k1'], params['k2'], params['p1'], params['p2'] = rest[:4]
  elif model == 'OPENCV_FISHEYE':
    params = dict(zip(['k1', 'k2', 'k3', 'k4'], rest[:4]))
    camtype = camera_utils.ProjectionType.FISHEYE
  return names, poses, pixtocam, params, camtype


def load_blender_posedata(data_dir, split=None):
  """`transforms[_split].json` as written by Blender / instant-ngp (datasets.py:152-186)."""
  suffix = '' if split is None else f'_{split}'
  with open(os.path.join(data_dir, f'transforms{suffix}.json'), 'r') as fp:
    meta = json.load(fp)
  names, poses = [], []
  for frame in meta['frames']:
    if os.path.exists(os.path.join(data_dir, frame['file_path'])):
      names.append(frame['file_path'].split('/')[-1])
      poses.append(np.array(frame['transform_matrix'], dtype=np.float32))
  poses = np.stack(poses, axis=0)
  w, h = meta['w'], meta['h']
  cx, cy = meta.get('cx', w / 2.), meta.get('cy', h / 2.)
  fx = meta['fl_x'] if 'fl_x' in meta else 0.5 * w / np.tan(0.5 * float(meta['camera_angle_x']))
  fy = meta['fl_y'] if 'fl_y' in meta else 0.5 * h / np.tan(0.5 * float(meta['camera_angle_y']))
  pixtocam = np.linalg.inv(camera_utils.intrinsic_matrix(fx, fy, cx, cy))
  coeffs = ['k1', 'k2', 'p1', 'p2']
  params = {c: meta.get(c, 0.) for c in coeffs} if any(c in meta for c in coeffs) else None
  return names, poses, pixtocam, params, camera_utils.ProjectionType.PERSPECTIVE


# ------------------------------------------------------------------------------------------ base class
class Dataset(threading.Thread, metaclass=abc.ABCMeta):
  """datasets.py:189-503.  A daemon thread keeps a queue of 3 host-side draws ahead of the consumer."""

  def __init__(self, split, data_dir, config, device=None, rank=0, world=1, start_thread=True):
    super().__init__()
    self._queue = queue.Queue(3)
    self.daemon = True
    self._patch_size = max(config.patch_size, 1)
    self._batch_size = config.batch_size // world
    if self._patch_size ** 2 > self._batch_size:
      raise ValueError(f'Patch size {self._patch_size}^2 too large for ' +
                       f'per-process batch size {self._batch_size}')
    self._batching = utils.BatchingMethod(config.batching)
    self._use_tiffs = config.use_tiffs
    self._load_disps = config.compute_disp_metrics
    self._load_normals = config.compute_normal_metrics
    self._test_camera_idx = 0
    self._num_border_pixels_to_mask = config.num_border_pixels_to_mask
    self._apply_bayer_mask = config.apply_bayer_mask
    self._cast_rays_in_train_step = config.cast_rays_in_train_step
    self._render_spherical = False
    self._rng = np.random.RandomState(20201473 + rank)          # train.py:45-47
    self.device = torch.device(device if device is not None else
                               ('cuda' if torch.cuda.is_available() else 'cpu'))

    self.split = utils.DataSplit(split)
    self.data_dir = data_dir
    self.near, self.far = config.near, config.far
    self.render_path = config.render_path
    self.distortion_params = None
    self.disp_images = self.normal_images = self.alphas = None
    self.poses = self.pixtocam_ndc = self.metadata = None
    self.camtype = camera_utils.ProjectionType.PERSPECTIVE
    self.exposures = self.render_exposures = None
    self.images = self.camtoworlds = self.pixtocams = None
    self.height = self.width = None

    self._load_renderings(config)

    if self.render_path:
      if config.render_path_file is not None:
        with open(config.render_path_file, 'rb') as fp:
          self.camtoworlds = np.load(fp)
      if config.render_resolution is not None:
        self.width, self.height = config.render_resolution
      if config.render_focal is not None:
        self.focal = config.render_focal
      if config.render_camtype is not None:
        if config.render_camtype == 'pano':
          self._render_spherical = True
        else:
          self.camtype = camera_utils.ProjectionType(config.render_camtype)
      self.distortion_params = None
      self.pixtocams = camera_utils.get_pixtocam(self.focal, self.width, self.height)

    self._n_examples = self.camtoworlds.shape[0]
    self.cameras = (self.pixtocams, self.camtoworlds, self.distortion_params, self.pixtocam_ndc)
    self._dev_cameras = None
    self._next_fn = self._next_train if self.split == utils.DataSplit.TRAIN else self._next_test
    self._queue.put(self._next_fn())       # seed the queue before the thread starts (no race on first use)
    if start_thread:
      self.start()

  # -------------------------------------------------------------------------- iterator protocol
  def __iter__(self):
    return self

  def __next__(self):
    """Next training batch or test example as a utils.Batch whose rays live on the device."""
    return self._finish(self._queue.get())

  def peek(self):
    """The next element without dequeuing it (datasets.py:372-383)."""
    return self._finish(copy.copy(self._queue.queue[0]))

  def run(self):
    while True:
      self._queue.put(self._next_fn())

  @property
  def size(self):
    return self._n_examples

  @abc.abstractmethod
  def _load_renderings(self, config):
    """Sets images [N,H,W,3], camtoworlds [N,3,4], pixtocams, height, width, focal (+ optional
    disp_images, normal_images, alphas, poses, distortion_params, metadata)."""

  # -------------------------------------------------------------------------- batches
  def device_cameras(self):
    if self._dev_cameras is None:
      t = lambda a: None if a is None else torch.as_tensor(np.asarray(a), dtype=torch.float32, device=self.device)
      self._dev_cameras = (t(self.pixtocams), t(self.camtoworlds), self.distortion_params, self.pixtocam_ndc)
    return self._dev_cameras

  def _make_pixel_batch(self, pix_x_int, pix_y_int, cam_idx, lossmult=None):
    """Host half of datasets.py:399-467: pixel coordinates + per-ray metadata + ground truth."""
    bc = lambda x: np.broadcast_to(x, pix_x_int.shape)[..., None]
    kw = {'lossmult': bc(1.).astype(np.float32) if lossmult is None else lossmult,
          'near': bc(self.near).astype(np.float32), 'far': bc(self.far).astype(np.float32),
          'cam_idx': bc(cam_idx).astype(np.int32)}
    if self.metadata is not None:
      for key in ['exposure_idx', 'exposure_values']:
        idx = 0 if self.render_path else cam_idx
        kw[key] = bc(self.metadata[key][idx])
    if self.exposures is not None:
      idx = 0 if self.render_path else cam_idx
      kw['exposure_values'] = bc(self.exposures[idx]).astype(np.float32)
    if self.render_path and self.render_exposures is not None:
      kw['exposure_values'] = bc(self.render_exposures[cam_idx]).astype(np.float32)
    pixels = utils.Pixels(np.broadcast_to(pix_x_int, pix_x_int.shape).astype(np.int32),
                          np.broadcast_to(pix_y_int, pix_x_int.shape).astype(np.int32), **kw)
    batch = {'rays': pixels}
    if not self.render_path:
      batch['rgb'] = self.images[cam_idx, pix_y_int, pix_x_int]
    if self._load_disps:
      batch['disps'] = self.disp_images[cam_idx, pix_y_int, pix_x_int]
    if self._load_normals:
      batch['normals'] = self.normal_images[cam_idx, pix_y_int, pix_x_int]
      batch['alphas'] = self.alphas[cam_idx, pix_y_int, pix_x_int]
    return utils.Batch(**batch)

  def _finish(self, batch):
    """Device half: pixels -> rays (one kernel launch), unless the train step does it itself.  A panorama's
    host item is its camera index alone: the whole panorama is cast on the device (datasets.py:488-492)."""
    if not isinstance(batch, utils.Batch):
      rays = camera_utils.cast_spherical_rays(self.camtoworlds[batch], self.height, self.width, self.near,
                                              self.far, device=self.device)
      return utils.Batch(rays=rays)
    if isinstance(batch.rays, utils.Rays):
      return batch
    if self._cast_rays_in_train_step and self.split == utils.DataSplit.TRAIN:
      return batch
    rays = camera_utils.cast_ray_batch(self.device_cameras(), batch.rays, self.camtype, device=self.device)
    return utils.Batch(rays=rays, rgb=batch.rgb, disps=batch.disps, normals=batch.normals, alphas=batch.alphas)

  def _next_train(self):
    """Random rays (datasets.py:469-503)."""
    num_patches = self._batch_size // self._patch_size ** 2
    lower = self._num_border_pixels_to_mask
    upper = self._num_border_pixels_to_mask + self._patch_size - 1
    pix_x = self._rng.randint(lower, self.width - upper, (num_patches, 1, 1))
    pix_y = self._rng.randint(lower, self.height - upper, (num_patches, 1, 1))
    dx, dy = camera_utils.pixel_coordinates(self._patch_size, self._patch_size)
    pix_x, pix_y = pix_x + dx, pix_y + dy
    if self._batching == utils.BatchingMethod.ALL_IMAGES:
      cam_idx = self._rng.randint(0, self._n_examples, (num_patches, 1, 1))
    else:
      cam_idx = self._rng.randint(0, self._n_examples, (1,))
    lossmult = None
    if self._apply_bayer_mask:
      from . import raw_utils
      lossmult = raw_utils.pixels_to_bayer_mask(pix_x, pix_y)
    return self._make_pixel_batch(pix_x, pix_y, cam_idx, lossmult=lossmult)

  def generate_ray_batch(self, cam_idx):
    """All pixels of one camera (datasets.py:505-517), rays on the device."""
    return self._finish(self._host_image_batch(cam_idx))

  def _host_image_batch(self, cam_idx):
    if self._render_spherical:
      return cam_idx
    pix_x, pix_y = camera_utils.pixel_coordinates(self.width, self.height)
    return self._make_pixel_batch(pix_x, pix_y, cam_idx)

  def _next_test(self):
    cam_idx = self._test_camera_idx
    self._test_camera_idx = (self._test_camera_idx + 1) % self._n_examples
    return self._host_image_batch(cam_idx)


# ------------------------------------------------------------------------------------------ loaders
class Blender(Dataset):
  """NeRF synthetic scenes: transforms_{split}.json + RGBA PNGs (datasets.py:507-560)."""

  def _load_renderings(self, config):
    if config.render_path:
      raise ValueError('render_path cannot be used for the blender dataset.')
    with open(os.path.join(self.data_dir, f'transforms_{self.split.value}.json'), 'r') as fp:
      meta = json.load(fp)
    images, disp_images, normal_images, cams = [], [], [], []
    for frame in meta['frames']:
      prefix = os.path.join(self.data_dir, frame['file_path'])

      def get_img(suffix, prefix=prefix):
        img = utils.load_img(prefix + suffix)
        return lib_image.downsample(img, config.factor) if config.factor > 1 else img
      if self._use_tiffs:
        img = lib_image.linear_to_srgb(np.stack([get_img(f'_{ch}.tiff') for ch in 'RGBA'], axis=-1))
      else:
        img = get_img('.png') / 255.
      images.append(img)
      if self._load_disps:
        disp_images.append(get_img('_disp.tiff'))
      if self._load_normals:
        normal_images.append(get_img('_normal.png')[..., :3] * 2. / 255. - 1.)
      cams.append(np.array(frame['transform_matrix'], dtype=np.float32))
    self.images = np.stack(images, axis=0)
    if self._load_disps:
      self.disp_images = np.stack(disp_images, axis=0)
    if self._load_normals:
      self.normal_images = np.stack(normal_images, axis=0)
      self.alphas = self.images[..., -1]
    rgb, alpha = self.images[..., :3], self.images[..., -1:]
    self.images = (rgb * alpha + (1. - alpha)).astype(np.float32)       # white background
    self.height, self.width = self.images.shape[1:3]
    self.camtoworlds = np.stack(cams, axis=0)
    self.focal = .5 * self.width / np.tan(.5 * float(meta['camera_angle_x']))
    self.pixtocams = camera_utils.get_pixtocam(self.focal, self.width, self.height)


class LLFF(Dataset):
  """Real captures posed by COLMAP (or a transforms.json): forward-facing (NDC) and 360 scenes, optional
  raw (RawNeRF) images (datasets.py:563-717)."""

  def _load_renderings(self, config):
    suffix, factor = '', 1
    if config.factor > 0 and not (config.rawnerf_mode and self.split == utils.DataSplit.TRAIN):
      suffix, factor = f'_{config.factor}', config.factor
    colmap_dir = os.path.join(self.data_dir, 'sparse/0/')
    if os.path.exists(colmap_dir):
      pose_data = load_colmap_posedata(colmap_dir)
    else:
      pose_data = load_blender_posedata(self.data_dir)
    image_names, poses, pixtocam, distortion_params, camtype = pose_data
    if config.load_alphabetical:
      order = np.argsort(image_names)
      image_names = [image_names[i] for i in order]
      poses = poses[order]
    self.pixtocams = (pixtocam @ np.diag([factor, factor, 1.])).astype(np.float32)
    self.focal = 1. / self.pixtocams[0, 0]
    self.distortion_params = distortion_params
    self.camtype = camtype

    raw_testscene = False
    if config.rawnerf_mode:
      from . import raw_utils
      images, metadata, raw_testscene = raw_utils.load_raw_dataset(
          self.split, self.data_dir, image_names, config.exposure_percentile, factor)
      self.metadata = metadata
    else:
      colmap_image_dir = os.path.join(self.data_dir, 'images')
      image_dir = os.path.join(self.data_dir, 'images' + suffix)
      for d in [image_dir, colmap_image_dir]:
        if not os.path.exists(d):
          raise ValueError(f'Image folder {d} does not exist.')
      # downsampled copies may be named differently: pair the two sorted listings
      colmap_to_image = dict(zip(sorted(os.listdir(colmap_image_dir)), sorted(os.listdir(image_dir))))
      images = np.stack([utils.load_img(os.path.join(image_dir, colmap_to_image[f])) for f in image_names],
                        axis=0) / 255.
      exifs = [utils.load_exif(os.path.join(colmap_image_dir, f)) for f in image_names]
      self.exifs = exifs
      if 'ExposureTime' in exifs[0] and 'ISOSpeedRatings' in exifs[0]:
        gather = lambda k: np.array([float(x[k]) for x in exifs])
        self.exposures = gather('ExposureTime') * gather('ISOSpeedRatings') / 1000.

    posefile = os.path.join(self.data_dir, 'poses_bounds.npy')
    if os.path.exists(posefile):
      bounds = np.load(posefile)[:, -2:]
    else:
      bounds = np.array([0.01, 1.])
    self.colmap_to_world_transform = np.eye(4)

    if config.forward_facing:
      self.pixtocam_ndc = self.pixtocams.reshape(-1, 3, 3)[0]
      scale = 1. / (bounds.min() * .75)
      poses[:, :3, 3] *= scale
      self.colmap_to_world_transform = np.diag([scale] * 3 + [1])
      bounds = bounds * scale
      poses, transform = camera_utils.recenter_poses(poses)
      self.colmap_to_world_transform = transform @ self.colmap_to_world_transform
      self.render_poses = camera_utils.generate_spiral_path(poses, bounds, n_frames=config.render_path_frames)
    else:
      poses, transform = camera_utils.transform_poses_pca(poses)
      self.colmap_to_world_transform = transform
      if config.render_spline_keyframes is not None:
        rets = camera_utils.create_render_spline_path(config, image_names, poses, self.exposures)
        self.spline_indices, self.render_poses, self.render_exposures = rets
      else:
        self.render_poses = camera_utils.generate_ellipse_path(
            poses, n_frames=config.render_path_frames, z_variation=config.z_variation, z_phase=config.z_phase)

    if raw_testscene:
      # the first COLMAP image shares the pose of the ground-truth test image; the rest are the training set
      poses = {utils.DataSplit.TEST: poses[:1], utils.DataSplit.TRAIN: poses[1:]}[self.split]
    self.poses = poses

    all_indices = np.arange(images.shape[0])
    if config.llff_use_all_images_for_training or raw_testscene:
      train_indices = all_indices
    else:
      train_indices = all_indices % config.llffhold != 0
    indices = {utils.DataSplit.TEST: all_indices[all_indices % config.llffhold == 0],
               utils.DataSplit.TRAIN: train_indices}[self.split]
    images = images[indices]
    poses = poses[indices]
    if self.exposures is not None:
      self.exposures = self.exposures[indices]
    if config.rawnerf_mode:
      for key in ['exposure_idx', 'exposure_values']:
        self.metadata[key] = self.metadata[key][indices]
    self.images = images.astype(np.float32)
    self.camtoworlds = self.render_poses if config.render_path else poses
    self.height, self.width = images.shape[1:3]


class TanksAndTemplesNerfPP(Dataset):
  """Tanks and Temples as processed by NeRF++ (datasets.py:720-764)."""

  def _load_renderings(self, config):
    basedir = os.path.join(self.data_dir, 'camera_path' if config.render_path else self.split.value)

    def load_files(dirname, load_fn, shape=None):
      files = [os.path.join(basedir, dirname, f) for f in sorted(os.listdir(os.path.join(basedir, dirname)))]
      mats = np.array([load_fn(f) for f in files])
      return mats.reshape(mats.shape[:1] + shape) if shape is not None else mats
    poses = load_files('pose', np.loadtxt, (4, 4)) @ np.diag([1., -1., -1., 1.])
    intrinsics = load_files('intrinsics', np.loadtxt, (4, 4))
    if not config.render_path:
      self.images = (load_files('rgb', utils.load_img) / 255.).astype(np.float32)
      self.height, self.width = self.images.shape[1:3]
    else:
      d = os.path.join(self.data_dir, 'test', 'rgb')
      self.height, self.width = utils.load_img(os.path.join(d, sorted(os.listdir(d))[0])).shape[:2]
      self.images = None
    self.camtoworlds = poses
    self.focal = intrinsics[0, 0, 0]
    self.pixtocams = camera_utils.get_pixtocam(self.focal, self.width, self.height)


class TanksAndTemplesFVS(Dataset):
  """Tanks and Temples as processed by Free View Synthesis (datasets.py:767-829)."""

  def _load_renderings(self, config):
    render_only = config.render_path and self.split == utils.DataSplit.TEST
    basedir = os.path.join(self.data_dir, 'dense')
    sizes = [f for f in sorted(os.listdir(basedir)) if f.startswith('ibr3d')][::-1]
    if config.factor >= len(sizes):
      raise ValueError(f'Factor {config.factor} larger than {len(sizes)}')
    basedir = os.path.join(basedir, sizes[config.factor])
    files = [f for f in sorted(os.listdir(basedir)) if f.startswith('im_')]
    if render_only:
      files = files[:1]
    images = np.array([utils.load_img(os.path.join(basedir, f)) for f in files]) / 255.
    intrinsics, rot, trans = (np.load(os.path.join(basedir, f'{n}.npy')) for n in ['Ks', 'Rs', 'ts'])
    w2c = np.concatenate([rot, trans[..., None]], axis=-1)
    c2w = np.linalg.inv(camera_utils.pad_poses(w2c))[:, :3, :4] @ np.diag([1., -1., -1., 1.])
    poses, _ = camera_utils.transform_poses_pca(c2w)            # z axis up
    self.poses = poses
    self.images = images.astype(np.float32)
    self.height, self.width = self.images.shape[1:3]
    self.camtoworlds = poses
    self.focal = intrinsics[0, 0, 0]
    self.pixtocams = camera_utils.get_pixtocam(self.focal, self.width, self.height)
    if render_only:
      path = camera_utils.generate_ellipse_path(poses, config.render_path_frames, z_variation=config.z_variation,
                                                z_phase=config.z_phase)
      self.images = None
      self.camtoworlds = self.render_poses = path
    else:
      idx = np.arange(images.shape[0])
      keep = idx[idx % config.llffhold == 0] if self.split == utils.DataSplit.TEST else idx[idx % config.llffhold != 0]
      self.images = self.images[keep]
      self.camtoworlds = self.camtoworlds[keep]


class DTU(Dataset):
  """DTU scans with the calibration files of `cal18` (datasets.py:832-911)."""

  def _load_renderings(self, config):
    if config.render_path:
      raise ValueError('render_path cannot be used for the DTU dataset.')
    import cv2
    light_cond = getattr(config, 'dtu_light_cond', 3)
    hold = getattr(config, 'dtuhold', 8)
    images, pixtocams, camtoworlds = [], [], []
    n_images = len(os.listdir(self.data_dir)) // 8            # 49 or 65 views, 8 light conditions each
    for i in range(1, n_images + 1):
      light = f'{light_cond}_r' + ('5000' if i < 50 else '7000') if light_cond < 7 else 'max'
      img = utils.load_img(os.path.join(self.data_dir, f'rect_{i:03d}_{light}.png')) / 255.
      if config.factor > 1:
        img = lib_image.downsample(img, config.factor)
      images.append(img)
      projection = np.loadtxt(os.path.join(self.data_dir, f'../../cal18/pos_{i:03d}.txt'), dtype=np.float32)
      cam, rot, t = cv2.decomposeProjectionMatrix(projection)[:3]
      cam = cam / cam[2, 2]
      pose = np.eye(4, dtype=np.float32)
      pose[:3, :3] = rot.transpose()
      pose[:3, 3] = (t[:3] / t[3])[:, 0]
      camtoworlds.append(pose[:3])
      if config.factor > 0:
        cam = np.diag([1. / config.factor, 1. / config.factor, 1.]).astype(np.float32) @ cam
      pixtocams.append(np.linalg.inv(cam))
    pixtocams, camtoworlds, images = np.stack(pixtocams), np.stack(camtoworlds), np.stack(images)
    camtoworlds, _ = camera_utils.recenter_poses(camtoworlds)
    camtoworlds = camtoworlds.copy()
    camtoworlds[:, :3, -1] /= np.max(np.abs(camtoworlds[:, :3, -1]))
    camtoworlds = camtoworlds @ np.diag([1., -1., -1., 1.]).astype(np.float32)     # OpenGL axes
    idx = np.arange(images.shape[0])
    keep = idx[idx % hold == 0] if self.split == utils.DataSplit.TEST else idx[idx % hold != 0]
    self.images = images[keep].astype(np.float32)
    self.height, self.width = images.shape[1:3]
    self.camtoworlds = camtoworlds[keep]
    self.pixtocams = pixtocams[keep]
