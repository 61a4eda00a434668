"""Rendering hand-off: batched `Camera` / `Physics.render` (reference: dm_control/mujoco/engine.py:178-233, 625-1100).

What the reference does through MuJoCo's OpenGL pipeline (mjv_updateScene + mjr_render on a GL context) becomes one
launch of a ray caster over the model's primitives (csrc/b200mj_render.cu, C ABI `b200mj_render`): B cameras, one per
environment, look at that environment's geoms and sites and produce `[B, H, W, 3]` uint8 rgb, `[B, H, W]` float32 depth
or `[B, H, W, 2]` int32 segmentation tensors that stay on the device (an observation for the task, or the hand-off to an
external renderer together with `scene_state()`).

Scope: depth and segmentation are geometric and follow the reference's definitions (distance along the optical axis,
engine.py:917-924; (object id, mjtObj) with -1 background, engine.py:926-944); `camera.matrix` is the reference's 3x4
camera matrix (engine.py:759-810). rgb is a headlight shade of `geom_rgba` — no textures, materials' reflectance,
shadows, skybox, overlays, scene callbacks or render flags: those need MuJoCo's GL renderer and stay out of scope.
"""
from __future__ import annotations

import collections
import ctypes

import numpy as np
import torch

from . import lib as _lib

OBJ_GEOM, OBJ_SITE = 5, 6      # mjtObj
_ZNEAR, _ZFAR = 0.01, 50.0     # mjModel.vis.map.znear / zfar defaults (fractions of stat.extent), engine.py:917-920

CameraMatrices = collections.namedtuple('CameraMatrices', ['image', 'focal', 'rotation', 'translation'])
Pose = collections.namedtuple('Pose', ['lookat', 'distance', 'azimuth', 'elevation'])


class _Scene(ctypes.Structure):
  _fields_ = [('nobj', ctypes.c_int), ('obj_type', ctypes.c_void_p), ('obj_kind', ctypes.c_void_p), ('obj_id', ctypes.c_void_p),
              ('visible', ctypes.c_void_p), ('rgba', ctypes.c_void_p), ('size', ctypes.c_void_p), ('size_stride', ctypes.c_longlong),
              ('pos', ctypes.c_void_p), ('mat', ctypes.c_void_p), ('cam_xpos', ctypes.c_void_p), ('cam_xmat', ctypes.c_void_p),
              ('fovy', ctypes.c_double), ('znear', ctypes.c_double), ('zfar', ctypes.c_double)]


def _quat_to_mat(q):
  w, x, y, z = q
  return np.array([[w*w + x*x - y*y - z*z, 2*(x*y - w*z), 2*(x*z + w*y)],
                   [2*(x*y + w*z), w*w - x*x + y*y - z*z, 2*(y*z - w*x)],
                   [2*(x*z - w*y), 2*(y*z + w*x), w*w - x*x - y*y + z*z]])


def _look_at(pos, target):
  """[B,3] camera positions, [B,3] targets -> [B,3,3] frames whose -z axis points at the target, x horizontal."""
  z = pos - target
  z = z / z.norm(dim=1, keepdim=True).clamp_min(1e-12)
  up = torch.zeros_like(z); up[:, 2] = 1.0
  x = torch.linalg.cross(up, z)
  degenerate = x.norm(dim=1, keepdim=True) < 1e-9
  x = torch.where(degenerate, torch.tensor([1.0, 0.0, 0.0], dtype=z.dtype, device=z.device).expand_as(x), x)
  x = x / x.norm(dim=1, keepdim=True)
  y = torch.linalg.cross(z, x)
  return torch.stack([x, y, z], dim=2)


class Camera:
  """B lock-stepped cameras, one per environment (reference: engine.Camera, engine.py:642-1000).

  `camera_id`: index or name of a model camera, or -1 for the free camera (engine.py:690-716), whose pose is the
  `MovableCamera` pose (lookat / distance / azimuth / elevation, engine.py:1003-1100) and can be changed with `set_pose`.
  """

  def __init__(self, physics, height=240, width=320, camera_id=-1, sites=True, groups=(0, 1, 2)):
    m = physics.model
    vis = getattr(m, 'vis', None)
    if not vis:
      raise ValueError('this model carries no visual tables (compiled before the rendering hand-off existed): recompile it')
    ncam = int(vis['cam_bodyid'].shape[0])
    if isinstance(camera_id, str):
      camera_id = m.name2id(camera_id, 'camera')
    if camera_id < -1:
      raise ValueError('camera_id cannot be smaller than -1.')
    if camera_id >= ncam:
      raise ValueError('model has {} fixed cameras. camera_id={} is invalid.'.format(ncam, camera_id))      # engine.py:700-703
    if height <= 0 or width <= 0:
      raise ValueError('image dimensions must be positive')
    self._physics, self._vis = physics, vis
    self.height, self.width, self.camera_id = int(height), int(width), int(camera_id)
    dev = physics.device
    d = physics.data
    for need in ('geom_xpos', 'geom_xmat', 'xpos', 'xmat'):
      if not hasattr(d, need):
        raise ValueError(f'rendering needs the `{need}` output: construct BatchedPhysics with outputs that include it')
    self._sites = bool(sites) and m.nsite > 0 and hasattr(d, 'site_xpos') and hasattr(d, 'site_xmat')
    ng, ns = m.ngeom, (m.nsite if self._sites else 0)
    self._nobj = ng + ns
    t32 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32), device=dev)
    self._type = t32(np.concatenate([m.geom_type, m.site_type[:ns]]))
    self._kind = t32(np.concatenate([np.full(ng, OBJ_GEOM), np.full(ns, OBJ_SITE)]))
    self._id = t32(np.concatenate([np.arange(ng), np.arange(ns)]))
    rgba = np.concatenate([vis['geom_rgba'].reshape(-1, 4), vis['site_rgba'].reshape(-1, 4)[:ns]]).astype(np.float32)
    group = np.concatenate([vis['geom_group'], vis['site_group'][:ns]])
    self._rgba = torch.as_tensor(rgba, device=dev).contiguous()
    self._visible = torch.as_tensor((np.isin(group, list(groups)) & (rgba[:, 3] > 0)).astype(np.uint8), device=dev)
    self._size_shared = torch.as_tensor(np.concatenate([m.geom_size, m.site_size[:ns]]).astype(np.float64),
                                        device=dev).contiguous()
    self._extent = float(vis['stat_extent'][0])
    self._free_pose = Pose(lookat=np.asarray(vis['stat_center'], dtype=np.float64).copy(), distance=1.5 * self._extent,
                           azimuth=90.0, elevation=-45.0)          # mjv_defaultFreeCamera
    self._fovy = float(vis['global_fovy'][0]) if camera_id == -1 else float(vis['cam_fovy'][camera_id])

  # ---- camera pose ----------------------------------------------------------------------------------------------
  def get_pose(self):
    if self.camera_id != -1:
      raise ValueError('only the free camera (camera_id=-1) has a settable pose')
    return self._free_pose

  def set_pose(self, lookat, distance, azimuth, elevation):
    """`MovableCamera.set_pose` (engine.py:1060-1085); the same pose for every environment."""
    if self.camera_id != -1:
      raise ValueError('only the free camera (camera_id=-1) has a settable pose')
    self._free_pose = Pose(np.asarray(lookat, dtype=np.float64).copy(), float(distance), float(azimuth), float(elevation))

  def pose(self):
    """-> cam_xpos [B,3], cam_xmat [B,3,3] (columns: right, up, backward) from the current body frames."""
    phys, vis, k = self._physics, self._vis, self.camera_id
    B, dev = phys.batch, phys.device
    f64 = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), device=dev)
    if k == -1:
      p = self._free_pose
      az, el = np.deg2rad(p.azimuth), np.deg2rad(p.elevation)
      forward = np.array([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)])
      pos = f64(p.lookat - p.distance * forward).expand(B, 3).contiguous()
      return pos, _look_at(pos, f64(p.lookat).expand(B, 3))
    d = phys.data
    b, mode = int(vis['cam_bodyid'][k]), int(vis['cam_mode'][k])
    xpos = d.xpos.reshape(B, -1, 3)[:, b]
    R = d.xmat.reshape(B, -1, 3, 3)[:, b]
    if mode == 0 or mode >= 3:
      pos = xpos + torch.matmul(R, f64(vis['cam_pos'][k]))
      mat = torch.matmul(R, f64(_quat_to_mat(vis['cam_quat'][k])))
      if mode >= 3:
        t = int(vis['cam_targetbodyid'][k])
        target = d.subtree_com.reshape(B, -1, 3)[:, t] if mode == 4 else d.xpos.reshape(B, -1, 3)[:, t]
        mat = _look_at(pos, target)
    elif mode == 1:
      pos, mat = xpos + f64(vis['cam_pos0'][k]), f64(vis['cam_mat0'][k]).reshape(3, 3).expand(B, 3, 3)
    else:
      pos = d.subtree_com.reshape(B, -1, 3)[:, b] + f64(vis['cam_poscom0'][k])
      mat = f64(vis['cam_mat0'][k]).reshape(3, 3).expand(B, 3, 3)
    return pos.contiguous(), mat.contiguous()

  def matrices(self):
    """`Camera.matrices` (engine.py:759-797), batched: image [3,3], focal [3,4], rotation [B,4,4], translation [B,4,4]."""
    pos, mat = self.pose()
    B, dev = pos.shape[0], pos.device
    translation = torch.eye(4, dtype=torch.float64, device=dev).repeat(B, 1, 1)
    translation[:, 0:3, 3] = -pos
    rotation = torch.eye(4, dtype=torch.float64, device=dev).repeat(B, 1, 1)
    rotation[:, 0:3, 0:3] = mat.transpose(1, 2)
    f = (1.0 / np.tan(np.deg2rad(self._fovy) / 2)) * self.height / 2.0
    focal = torch.as_tensor(np.diag([-f, f, 1.0, 0])[0:3, :], device=dev)
    image = torch.eye(3, dtype=torch.float64, device=dev)
    image[0, 2] = (self.width - 1) / 2.0
    image[1, 2] = (self.height - 1) / 2.0
    return CameraMatrices(image=image, focal=focal, rotation=rotation, translation=translation)

  @property
  def matrix(self):
    """The 3x4 camera matrix of every environment, [B,3,4] (engine.py:799-810)."""
    image, focal, rotation, translation = self.matrices()
    return image @ focal @ rotation @ translation

  # ---- images ---------------------------------------------------------------------------------------------------
  def _sizes(self):
    """object sizes: shared [nobj,3], or [B,nobj,3] when the model has per-environment geoms (corridor walls)."""
    phys = self._physics
    var = getattr(phys, '_var_geom_ids', None)
    if var is None or len(var) == 0:
      return self._size_shared, 0
    B = phys.batch
    s = self._size_shared.expand(B, -1, -1).clone()
    s[:, torch.as_tensor(np.asarray(var, dtype=np.int64), device=s.device)] = phys.data.var_geom_size.reshape(B, -1, 3)
    return s.contiguous(), self._nobj * 3

  def render(self, depth=False, segmentation=False):
    """-> [B,H,W,3] uint8 | [B,H,W] float32 (depth) | [B,H,W,2] int32 (segmentation). `Camera.render`, engine.py:840-946."""
    if depth and segmentation:
      raise ValueError('Only one of depth or segmentation can be True at once.')      # engine.py:869-870
    phys = self._physics
    if phys.is_dirty:          # state written through a binding since the last forward / step (mjcf/physics.py:225-237)
      phys.forward()
    d, B, dev = phys.data, phys.batch, phys.device
    ng = phys.model.ngeom
    if self._sites:
      pos = torch.cat([d.geom_xpos.reshape(B, ng, 3), d.site_xpos.reshape(B, -1, 3)], dim=1).contiguous()
      mat = torch.cat([d.geom_xmat.reshape(B, ng, 9), d.site_xmat.reshape(B, -1, 9)], dim=1).contiguous()
    else:
      pos, mat = d.geom_xpos.reshape(B, ng, 3).contiguous(), d.geom_xmat.reshape(B, ng, 9).contiguous()
    cam_pos, cam_mat = self.pose()
    cam_mat = cam_mat.reshape(B, 9).contiguous()
    size, stride = self._sizes()
    H, W = self.height, self.width
    rgb = dep = seg = None
    if depth:
      dep = torch.empty(B, H, W, dtype=torch.float32, device=dev)
    elif segmentation:
      seg = torch.empty(B, H, W, 2, dtype=torch.int32, device=dev)
    else:
      rgb = torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev)
    ptr = lambda t: None if t is None else t.data_ptr()
    sc = _Scene(self._nobj, ptr(self._type), ptr(self._kind), ptr(self._id), ptr(self._visible), ptr(self._rgba), ptr(size), stride,
                ptr(pos), ptr(mat), ptr(cam_pos), ptr(cam_mat), self._fovy, _ZNEAR * self._extent, _ZFAR * self._extent)
    L = _lib.load()
    with torch.cuda.device(dev):
      _lib.check(L.b200mj_render(ctypes.byref(sc), B, H, W, ptr(rgb), ptr(dep), ptr(seg),
                                 ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return dep if depth else (seg if segmentation else rgb)


def scene_state(physics, env_ids=None):
  """Host copies of what an external renderer needs for the chosen environments: MuJoCo-named numpy arrays
  (`geom_xpos`, `geom_xmat`, `geom_size`, `geom_type`, `geom_rgba`, site_*, and `cam_xpos` / `cam_xmat` of every model camera)."""
  m, d, B = physics.model, physics.data, physics.batch
  idx = torch.arange(B, device=physics.device) if env_ids is None else torch.as_tensor(env_ids, device=physics.device)
  take = lambda t, shape: t.index_select(0, idx).reshape((len(idx),) + shape).cpu().numpy()
  out = dict(geom_type=np.asarray(m.geom_type), geom_size=np.asarray(m.geom_size), geom_rgba=m.vis['geom_rgba'],
             geom_xpos=take(d.geom_xpos, (m.ngeom, 3)), geom_xmat=take(d.geom_xmat, (m.ngeom, 9)))
  if m.nsite and hasattr(d, 'site_xpos'):
    out.update(site_type=np.asarray(m.site_type), site_size=np.asarray(m.site_size), site_rgba=m.vis['site_rgba'],
               site_xpos=take(d.site_xpos, (m.nsite, 3)), site_xmat=take(d.site_xmat, (m.nsite, 9)))
  ncam = int(m.vis['cam_bodyid'].shape[0])
  if ncam:
    poses = [Camera(physics, 1, 1, k).pose() for k in range(ncam)]
    out['cam_xpos'] = torch.stack([p for p, _ in poses], 1).index_select(0, idx).cpu().numpy()
    out['cam_xmat'] = torch.stack([r.reshape(B, 9) for _, r in poses], 1).index_select(0, idx).cpu().numpy()
  return out
