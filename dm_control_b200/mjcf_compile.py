"""MJCF-subset compiler: XML -> compiled `Model` tables (host side, one-time per model).

The reference has no compiler of its own: `dm_control/mujoco/wrapper/core.py:179-182` hands the XML
string to `mujoco.MjModel.from_xml_string` (the un-vendored MuJoCo C++ compiler). This module restates
the subset of MuJoCo's documented compile semantics that the hot-path configs need
(`dm_control/suite/{cartpole,cheetah,humanoid,quadruped}.xml`, `suite/common/*.xml`,
`locomotion/walkers/assets/humanoid_CMU_V2019.xml`): includes, nested default classes + childclass,
`<compiler angle/eulerseq/settotalmass/inertiafromgeom>`, `<option>` + flags, body tree with
pos/quat/euler/axisangle/xyaxes/zaxis frames, free/ball/slide/hinge joints, plane/sphere/capsule/
ellipsoid/cylinder/box geoms incl. `fromto`, sites, `<inertial>`, motor/general/position/velocity
actuators, fixed tendons, joint/tendon equalities, contact excludes, the sensor kinds listed in
include/b200mj_model_fields.h, keyframes (qpos), and the derived constants MuJoCo computes in
`mj_setConst` (`*_invweight0`, `meaninertia`, `tendon_length0`, subtree masses).

Nothing here runs per step; it is numpy on purpose.
"""
from __future__ import annotations

import math
import os
import xml.etree.ElementTree as ET

import numpy as np

from . import model as _model

# ---------------------------------------------------------------------------------------------
# small math
# ---------------------------------------------------------------------------------------------

def _floats(s, n=None):
  v = np.array([float(x) for x in str(s).replace(',', ' ').split()], dtype=np.float64)
  if n is not None and v.size != n:
    raise ValueError(f'expected {n} numbers, got {s!r}')
  return v


def quat_mul(a, b):
  return np.array([
      a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
      a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
      a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
      a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def quat_conj(q):
  return np.array([q[0], -q[1], -q[2], -q[3]])


def quat_to_mat(q):
  w, x, y, z = q
  return np.array([
      [w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
      [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
      [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


def mat_to_quat(m):
  """Rotation matrix -> unit quaternion (w,x,y,z), w >= 0 branch preferred."""
  t = np.trace(m)
  if t > 0:
    s = math.sqrt(t + 1.0) * 2
    q = np.array([0.25 * s, (m[2, 1] - m[1, 2]) / s, (m[0, 2] - m[2, 0]) / s, (m[1, 0] - m[0, 1]) / s])
  elif m[0, 0] > m[1, 1] and m[0, 0] > m[2, 2]:
    s = math.sqrt(1.0 + m[0, 0] - m[1, 1] - m[2, 2]) * 2
    q = np.array([(m[2, 1] - m[1, 2]) / s, 0.25 * s, (m[0, 1] + m[1, 0]) / s, (m[0, 2] + m[2, 0]) / s])
  elif m[1, 1] > m[2, 2]:
    s = math.sqrt(1.0 + m[1, 1] - m[0, 0] - m[2, 2]) * 2
    q = np.array([(m[0, 2] - m[2, 0]) / s, (m[0, 1] + m[1, 0]) / s, 0.25 * s, (m[1, 2] + m[2, 1]) / s])
  else:
    s = math.sqrt(1.0 + m[2, 2] - m[0, 0] - m[1, 1]) * 2
    q = np.array([(m[1, 0] - m[0, 1]) / s, (m[0, 2] + m[2, 0]) / s, (m[1, 2] + m[2, 1]) / s, 0.25 * s])
  q = q / np.linalg.norm(q)
  if q[0] < 0:
    q = -q
  return q


def axisangle_to_quat(axis, angle):
  axis = np.asarray(axis, dtype=np.float64)
  n = np.linalg.norm(axis)
  if n < 1e-14:
    return np.array([1.0, 0, 0, 0])
  axis = axis / n
  return np.concatenate([[math.cos(angle / 2)], axis * math.sin(angle / 2)])


def z_to_quat(vec):
  """Quaternion rotating (0,0,1) onto `vec` (MuJoCo's zaxis / fromto convention)."""
  vec = np.asarray(vec, dtype=np.float64)
  vec = vec / np.linalg.norm(vec)
  axis = np.cross([0.0, 0.0, 1.0], vec)
  s = np.linalg.norm(axis)
  if s < 1e-10:
    axis = np.array([1.0, 0.0, 0.0])
  else:
    axis = axis / s
  ang = math.atan2(s, vec[2])
  return np.concatenate([[math.cos(ang / 2)], axis * math.sin(ang / 2)])


def rot_vec(q, v):
  return quat_to_mat(q) @ np.asarray(v, dtype=np.float64)


# ---------------------------------------------------------------------------------------------
# XML loading: includes + defaults
# ---------------------------------------------------------------------------------------------

def _expand_includes(root, base_dir, assets):
  """Replace every <include file=.../> by the children of the included file's root, in place."""
  changed = True
  while changed:
    changed = False
    for parent in list(root.iter()):
      for idx, child in enumerate(list(parent)):
        if child.tag != 'include':
          continue
        fname = child.attrib['file']
        text = None
        if assets:
          for key in (fname, os.path.basename(fname), fname.lstrip('./')):
            if key in assets:
              text = assets[key]
              break
        if text is None:
          path = fname if os.path.isabs(fname) else os.path.join(base_dir or '.', fname)
          with open(path, 'rb') as f:
            text = f.read()
        if isinstance(text, bytes):
          text = text.decode('utf-8')
        inc = ET.fromstring(text)
        pos = list(parent).index(child)
        parent.remove(child)
        for k, sub in enumerate(list(inc)):
          parent.insert(pos + k, sub)
        changed = True


_ACTUATOR_TAGS = ('general', 'motor', 'position', 'velocity', 'intvelocity', 'damper', 'cylinder', 'muscle',
                  'adhesion')
_DEFAULT_TAGS = ('geom', 'joint', 'site', 'equality', 'tendon', 'camera', 'light', 'material', 'mesh', 'pair')


class _Defaults:
  """Tree of <default class=...> nodes. Each node maps tag -> merged attribute dict."""

  def __init__(self):
    self.classes = {}

  def build(self, root):
    self.classes['main'] = {}
    for d in root.findall('default'):
      self._walk(d, None, top=True)

  def _walk(self, node, parent_name, top=False):
    # MuJoCo reads a <default> in two passes: its own element children first, nested classes second,
    # so a nested class inherits the parent's final attribute set.
    if top:
      name = 'main'
      cur = self.classes['main']
    else:
      name = node.attrib.get('class')
      if name is None:
        raise ValueError('nested <default> needs a class name')
      cur = {k: dict(v) for k, v in self.classes[parent_name].items()}
    for child in node:
      if child.tag == 'default':
        continue
      tag = 'general' if child.tag in _ACTUATOR_TAGS else child.tag
      entry = cur.setdefault(tag, {})
      if child.tag in _ACTUATOR_TAGS and child.tag != 'general':
        entry.update(_actuator_shortcut(child.tag, child.attrib, entry))
      else:
        entry.update(child.attrib)
    self.classes[name] = cur
    for child in node:
      if child.tag == 'default':
        self._walk(child, name)

  def get(self, tag, cls):
    return dict(self.classes.get(cls or 'main', self.classes['main']).get(tag, {}))


def _actuator_shortcut(tag, attrib, inherited=None):
  """Expand <motor>/<position>/<velocity> shortcut attributes into <general> attributes."""
  out = dict(attrib)
  if tag == 'motor':
    out.update(dyntype='none', gaintype='fixed', biastype='none', gainprm='1', biasprm='0 0 0')
  elif tag == 'position':
    kp = float(out.pop('kp', (inherited or {}).get('_kp', 1.0)))
    kv = float(out.pop('kv', (inherited or {}).get('_kv', 0.0)))
    out.update(dyntype='none', gaintype='fixed', biastype='affine', gainprm=f'{kp!r}',
               biasprm=f'0 {-kp!r} {-kv!r}', _kp=kp, _kv=kv)
  elif tag == 'velocity':
    kv = float(out.pop('kv', (inherited or {}).get('_kv', 1.0)))
    out.update(dyntype='none', gaintype='fixed', biastype='affine', gainprm=f'{kv!r}', biasprm=f'0 0 {-kv!r}',
               _kv=kv)
  elif tag == 'general':
    pass
  else:
    raise NotImplementedError(f'actuator shortcut <{tag}> is outside the supported MJCF subset')
  return out


# ---------------------------------------------------------------------------------------------
# geometry: mass / inertia of primitive geoms
# ---------------------------------------------------------------------------------------------

_GEOM_TYPES = {'plane': 0, 'hfield': 1, 'sphere': 2, 'capsule': 3, 'ellipsoid': 4, 'cylinder': 5, 'box': 6,
               'mesh': 7}
_JNT_TYPES = {'free': 0, 'ball': 1, 'slide': 2, 'hinge': 3}


def _geom_volume_inertia(gtype, size):
  """Volume and unit-density diagonal inertia (about the geom centre, geom frame)."""
  if gtype == 2:  # sphere
    r = size[0]
    v = 4.0 / 3.0 * math.pi * r ** 3
    i = 0.4 * v * r * r
    return v, np.array([i, i, i])
  if gtype == 3:  # capsule: cylinder + two half spheres
    r, h = size[0], size[1]
    height = 2 * h
    vc = math.pi * r * r * height
    vs = 4.0 / 3.0 * math.pi * r ** 3
    ixx = vc * (3 * r * r + height * height) / 12.0 + vs * (0.4 * r * r + 0.375 * r * height + 0.25 * height * height)
    izz = vc * r * r / 2.0 + vs * 0.4 * r * r
    return vc + vs, np.array([ixx, ixx, izz])
  if gtype == 4:  # ellipsoid
    a, b, c = size
    v = 4.0 / 3.0 * math.pi * a * b * c
    return v, v / 5.0 * np.array([b * b + c * c, a * a + c * c, a * a + b * b])
  if gtype == 5:  # cylinder
    r, h = size[0], size[1]
    height = 2 * h
    v = math.pi * r * r * height
    ixx = v * (3 * r * r + height * height) / 12.0
    return v, np.array([ixx, ixx, v * r * r / 2.0])
  if gtype == 6:  # box
    a, b, c = size
    v = 8 * a * b * c
    return v, v / 3.0 * np.array([b * b + c * c, a * a + c * c, a * a + b * b])
  return 0.0, np.zeros(3)


def _geom_rbound(gtype, size):
  if gtype == 2:
    return size[0]
  if gtype == 3:
    return size[0] + size[1]
  if gtype == 4:
    return max(size)
  if gtype == 5:
    return math.sqrt(size[0] ** 2 + size[1] ** 2)
  if gtype == 6:
    return float(np.linalg.norm(size))
  return 0.0


# ---------------------------------------------------------------------------------------------
# the compiler
# ---------------------------------------------------------------------------------------------

class _Compiler:

  def __init__(self, root, base_dir, assets):
    self.root = root
    _expand_includes(root, base_dir, assets)
    self.defaults = _Defaults()
    self.defaults.build(root)
    comp = {}
    for c in root.findall('compiler'):
      comp.update(c.attrib)
    self.degree = comp.get('angle', 'degree') == 'degree'
    self.eulerseq = comp.get('eulerseq', 'xyz')
    self.settotalmass = float(comp.get('settotalmass', -1))
    self.inertiafromgeom = comp.get('inertiafromgeom', 'auto')
    self.autolimits = comp.get('autolimits', 'true') == 'true'
    self.boundmass = float(comp.get('boundmass', 0))
    self.boundinertia = float(comp.get('boundinertia', 0))
    if comp.get('coordinate', 'local') != 'local':
      raise NotImplementedError('global coordinates are outside the supported MJCF subset')
    # element lists
    self.bodies = []   # dicts
    self.joints = []
    self.geoms = []
    self.sites = []
    self.cameras = []
    self.names = {k: {} for k in ('body', 'joint', 'geom', 'site', 'actuator', 'tendon', 'sensor', 'equality',
                                  'key', 'camera')}
    # visual-only tables (rendering hand-off, dm_control_b200/render.py): material colours; they never reach the physics blob
    self.material_rgba = {}
    self.materials, self.textures, self.lights = [], [], []      # (name or placeholder) per element, in document order
    for asset in root.findall('asset'):
      for mat in asset.findall('material'):
        a = self.defaults.get('material', mat.attrib.get('class'))
        a.update(mat.attrib)
        name = a.get('name', f'_material{len(self.materials)}')
        self.materials.append(name)
        self.material_rgba[name] = _floats(a.get('rgba', '1 1 1 1'), 4)
      for tex in asset.findall('texture'):
        self.textures.append(tex.attrib.get('name', f'_texture{len(self.textures)}'))
    self.custom = {k: [e.attrib.get('name', f'_{k}{i}') for i, e in enumerate(e for cu in root.findall('custom') for e in cu.findall(k))]
                   for k in ('numeric', 'text', 'tuple')}

  # ---- attribute helpers -------------------------------------------------------------------
  def _merged(self, tag, elem, childclass):
    cls = elem.attrib.get('class', childclass)
    a = self.defaults.get(tag, cls)
    a.update(elem.attrib)
    return a

  def _angle(self, x):
    return np.asarray(x, dtype=np.float64) * (math.pi / 180.0 if self.degree else 1.0)

  def _frame_quat(self, a):
    """Orientation from quat / axisangle / euler / xyaxes / zaxis attributes (MuJoCo frame orientations)."""
    if 'quat' in a:
      q = _floats(a['quat'], 4)
      return q / np.linalg.norm(q)
    if 'axisangle' in a:
      v = _floats(a['axisangle'], 4)
      return axisangle_to_quat(v[:3], float(self._angle(v[3])))
    if 'euler' in a:
      e = self._angle(_floats(a['euler'], 3))
      q = np.array([1.0, 0, 0, 0])
      for ch, ang in zip(self.eulerseq, e):
        ax = {'x': [1.0, 0, 0], 'y': [0, 1.0, 0], 'z': [0, 0, 1.0]}[ch.lower()]
        r = axisangle_to_quat(ax, float(ang))
        q = quat_mul(q, r) if ch.islower() else quat_mul(r, q)
      return q / np.linalg.norm(q)
    if 'xyaxes' in a:
      v = _floats(a['xyaxes'], 6)
      x = v[:3] / np.linalg.norm(v[:3])
      y = v[3:] - x * np.dot(x, v[3:])
      y = y / np.linalg.norm(y)
      z = np.cross(x, y)
      return mat_to_quat(np.stack([x, y, z], axis=1))
    if 'zaxis' in a:
      return z_to_quat(_floats(a['zaxis'], 3))
    return np.array([1.0, 0, 0, 0])

  # ---- tree walk ---------------------------------------------------------------------------
  def walk(self):
    world = self.root.find('worldbody')
    self.bodies.append(dict(name='world', parent=0, pos=np.zeros(3), quat=np.array([1.0, 0, 0, 0]),
                            inertial=None, depth=0))
    self.names['body']['world'] = 0
    if world is not None:
      self._body_children(world, 0, None)

  def _body_children(self, elem, bid, childclass):
    for child in elem:
      if child.tag == 'geom':
        self._add_geom(child, bid, childclass)
      elif child.tag in ('joint', 'freejoint'):
        self._add_joint(child, bid, childclass)
      elif child.tag == 'site':
        self._add_site(child, bid, childclass)
      elif child.tag == 'camera':
        self._add_camera(child, bid, childclass)
      elif child.tag == 'light':
        self.lights.append(child.attrib.get('name', f'_light{len(self.lights)}'))
      elif child.tag == 'inertial':
        a = child.attrib
        inert = dict(pos=_floats(a['pos'], 3), quat=self._frame_quat(a), mass=float(a['mass']))
        if 'diaginertia' in a:
          inert['diag'] = _floats(a['diaginertia'], 3)
        elif 'fullinertia' in a:
          f = _floats(a['fullinertia'], 6)
          full = np.array([[f[0], f[3], f[4]], [f[3], f[1], f[5]], [f[4], f[5], f[2]]])
          w, v = np.linalg.eigh(full)
          order = np.argsort(-w)
          v = v[:, order]
          if np.linalg.det(v) < 0:
            v[:, 2] = -v[:, 2]
          inert['diag'] = w[order]
          inert['quat'] = quat_mul(inert['quat'], mat_to_quat(v))
        self.bodies[bid]['inertial'] = inert
    for child in elem:
      if child.tag == 'body':
        a = child.attrib
        cc = a.get('childclass', childclass)
        nb = len(self.bodies)
        name = a.get('name', f'_body{nb}')
        self.bodies.append(dict(name=name, parent=bid, pos=_floats(a.get('pos', '0 0 0'), 3),
                                quat=self._frame_quat(a), inertial=None,
                                depth=self.bodies[bid]['depth'] + 1, mocap=a.get('mocap', 'false') == 'true'))
        self.names['body'][name] = nb
        self._body_children(child, nb, cc)

  def _add_joint(self, elem, bid, childclass):
    if elem.tag == 'freejoint':
      a = dict(elem.attrib)
      a['type'] = 'free'
      # freejoint ignores defaults entirely (MuJoCo XML reference, body/freejoint)
      a.setdefault('limited', 'false')
      a.update(stiffness='0', damping='0', armature='0', frictionloss='0')
    else:
      a = self._merged('joint', elem, childclass)
    jtype = _JNT_TYPES[a.get('type', 'hinge')]
    name = a.get('name', f'_joint{len(self.joints)}')
    rng = _floats(a.get('range', '0 0'), 2)
    if jtype in (1, 3):
      rng = self._angle(rng)
    limited = a.get('limited', 'auto')
    if limited == 'auto':
      limited = self.autolimits and ('range' in a)
    else:
      limited = limited == 'true'
    axis = _floats(a.get('axis', '0 0 1'), 3)
    if jtype in (2, 3):
      axis = axis / np.linalg.norm(axis)
    ref = float(a.get('ref', 0))
    springref = float(a.get('springref', 0))
    if jtype == 3:
      ref = float(self._angle(ref))
      springref = float(self._angle(springref))
    j = dict(name=name, body=bid, type=jtype, pos=_floats(a.get('pos', '0 0 0'), 3), axis=axis,
             stiffness=float(a.get('stiffness', 0)), damping=float(a.get('damping', 0)),
             armature=float(a.get('armature', 0)), frictionloss=float(a.get('frictionloss', 0)),
             limited=bool(limited), range=rng, margin=float(a.get('margin', 0)), ref=ref, springref=springref,
             solref=_floats(a.get('solreflimit', '0.02 1'), 2), solimp=_solimp(a.get('solimplimit')),
             solreffriction=_floats(a.get('solreffriction', '0.02 1'), 2),
             solimpfriction=_solimp(a.get('solimpfriction')))
    self.names['joint'][name] = len(self.joints)
    self.joints.append(j)

  def _add_geom(self, elem, bid, childclass):
    a = self._merged('geom', elem, childclass)
    gtype = _GEOM_TYPES[a.get('type', 'sphere')]
    if gtype in (1, 7):
      raise NotImplementedError('hfield/mesh geoms are outside the supported MJCF subset')
    size = np.zeros(3)
    if 'size' in a:
      s = _floats(a['size'])
      size[:s.size] = s[:3]
    pos = _floats(a.get('pos', '0 0 0'), 3)
    quat = self._frame_quat(a)
    if 'fromto' in a:
      ft = _floats(a['fromto'], 6)
      p0, p1 = ft[:3], ft[3:]
      pos = 0.5 * (p0 + p1)
      vec = p1 - p0  # MuJoCo aligns +z with (to - from)
      half = 0.5 * np.linalg.norm(vec)
      quat = z_to_quat(vec)
      if gtype in (3, 5):
        size[1] = half
      elif gtype in (4, 6):
        size[2] = half
    name = a.get('name', f'_geom{len(self.geoms)}')
    g = dict(name=name, body=bid, type=gtype, size=size, pos=pos, quat=quat,
             condim=int(a.get('condim', 3)), contype=int(a.get('contype', 1)),
             conaffinity=int(a.get('conaffinity', 1)), priority=int(a.get('priority', 0)),
             friction=_pad(_floats(a.get('friction', '1 0.005 0.0001')), [1, 0.005, 0.0001]),
             solmix=float(a.get('solmix', 1)), solref=_floats(a.get('solref', '0.02 1'), 2),
             solimp=_solimp(a.get('solimp')), margin=float(a.get('margin', 0)), gap=float(a.get('gap', 0)),
             density=float(a.get('density', 1000)), mass=(float(a['mass']) if 'mass' in a else None),
             rgba=self._rgba(a), group=int(a.get('group', 0)))
    self.names['geom'][name] = len(self.geoms)
    self.geoms.append(g)

  def _add_site(self, elem, bid, childclass):
    a = self._merged('site', elem, childclass)
    stype = _GEOM_TYPES[a.get('type', 'sphere')]
    size = np.full(3, 0.005)
    if 'size' in a:
      s = _floats(a['size'])
      size[:s.size] = s[:3]
    pos = _floats(a.get('pos', '0 0 0'), 3)
    quat = self._frame_quat(a)
    if 'fromto' in a:
      ft = _floats(a['fromto'], 6)
      pos = 0.5 * (ft[:3] + ft[3:])
      vec = ft[3:] - ft[:3]
      quat = z_to_quat(vec)
      if stype in (3, 5):
        size[1] = 0.5 * np.linalg.norm(vec)
      else:
        size[2] = 0.5 * np.linalg.norm(vec)
    name = a.get('name', f'_site{len(self.sites)}')
    self.names['site'][name] = len(self.sites)
    self.sites.append(dict(name=name, body=bid, type=stype, size=size, pos=pos, quat=quat, rgba=self._rgba(a),
                           group=int(a.get('group', 0))))

  def _rgba(self, a):
    # explicit rgba wins; else the material's colour; else MuJoCo's default grey
    if 'rgba' in a:
      return _floats(a['rgba'], 4)
    if a.get('material') in self.material_rgba:
      return self.material_rgba[a['material']].copy()
    return np.array([0.5, 0.5, 0.5, 1.0])

  def _add_camera(self, elem, bid, childclass):
    """<camera>: pose in the body frame, vertical field of view, tracking mode (MuJoCo XML reference, body/camera)."""
    a = self._merged('camera', elem, childclass)
    name = a.get('name', f'_camera{len(self.cameras)}')
    mode = {'fixed': 0, 'track': 1, 'trackcom': 2, 'targetbody': 3, 'targetbodycom': 4}[a.get('mode', 'fixed')]
    self.names['camera'][name] = len(self.cameras)
    self.cameras.append(dict(name=name, body=bid, pos=_floats(a.get('pos', '0 0 0'), 3), quat=self._frame_quat(a), mode=mode,
                             fovy=(float(a['fovy']) if 'fovy' in a else None), target=a.get('target')))


def _pad(v, default):
  out = np.array(default, dtype=np.float64)
  out[:v.size] = v[:out.size]
  return out


def _solimp(s):
  return _pad(_floats(s), [0.9, 0.95, 0.001, 0.5, 2]) if s is not None else np.array([0.9, 0.95, 0.001, 0.5, 2])


_DISABLE_BITS = dict(constraint=1 << 0, equality=1 << 1, frictionloss=1 << 2, limit=1 << 3, contact=1 << 4,
                     passive=1 << 5, gravity=1 << 6, clampctrl=1 << 7, warmstart=1 << 8, filterparent=1 << 9,
                     actuation=1 << 10, refsafe=1 << 11, sensor=1 << 12, midphase=1 << 13, eulerdamp=1 << 14)
_ENABLE_BITS = dict(override=1 << 0, energy=1 << 1, fwdinv=1 << 2, invdiscrete=1 << 3, multiccd=1 << 4,
                    island=1 << 5)

_SENSOR_KINDS = {
    # tag: (type id, objtype tag attr, dim, needstage 1=pos 2=vel 3=acc)
    'touch': (0, 'site', 1, 3), 'accelerometer': (1, 'site', 3, 3), 'velocimeter': (2, 'site', 3, 2),
    'gyro': (3, 'site', 3, 2), 'force': (4, 'site', 3, 3), 'torque': (5, 'site', 3, 3),
    'jointpos': (8, 'joint', 1, 1), 'jointvel': (9, 'joint', 1, 2), 'actuatorfrc': (14, 'actuator', 1, 3),
    'framepos': (25, None, 3, 1), 'subtreecom': (34, 'body', 3, 1), 'subtreelinvel': (35, 'body', 3, 2),
    'subtreeangmom': (36, 'body', 3, 2)}
_OBJ = dict(body=1, xbody=2, joint=3, geom=5, site=6, actuator=19)


def compile_xml(xml, assets=None, base_dir=None, nconmax=None, njmax=None):
  """Compile an MJCF string (or bytes) into a `dm_control_b200.model.Model`."""
  if isinstance(xml, bytes):
    xml = xml.decode('utf-8')
  root = ET.fromstring(xml)
  c = _Compiler(root, base_dir, assets)
  c.walk()
  return _finish(c, root, nconmax, njmax)


def compile_file(path, assets=None, **kw):
  with open(path, 'rb') as f:
    return compile_xml(f.read(), assets=assets, base_dir=os.path.dirname(os.path.abspath(path)), **kw)


def _finish(c, root, nconmax, njmax):
  F = {}
  nbody, njnt, ngeom, nsite = len(c.bodies), len(c.joints), len(c.geoms), len(c.sites)

  # ---- options ----------------------------------------------------------------------------
  opt = {}
  flags_dis, flags_en = 0, 0
  for o in root.findall('option'):
    opt.update(o.attrib)
    for fl in o.findall('flag'):
      for k, v in fl.attrib.items():
        if k in _DISABLE_BITS:
          flags_dis = (flags_dis | _DISABLE_BITS[k]) if v == 'disable' else (flags_dis & ~_DISABLE_BITS[k])
        elif k in _ENABLE_BITS:
          flags_en = (flags_en | _ENABLE_BITS[k]) if v == 'enable' else (flags_en & ~_ENABLE_BITS[k])
  integrator = {'Euler': 0, 'RK4': 1, 'implicit': 2, 'implicitfast': 3}[opt.get('integrator', 'Euler')]
  solver = {'PGS': 0, 'CG': 1, 'Newton': 2}[opt.get('solver', 'Newton')]
  cone = {'pyramidal': 0, 'elliptic': 1}[opt.get('cone', 'pyramidal')]
  if cone != 0:
    raise NotImplementedError('elliptic cones are outside the supported subset')
  gravity = _floats(opt.get('gravity', '0 0 -9.81'), 3)
  timestep = float(opt.get('timestep', 0.002))

  # ---- bodies, joints, dofs ---------------------------------------------------------------
  body_parent = np.array([b['parent'] for b in c.bodies], dtype=np.int32)
  body_jntnum = np.zeros(nbody, np.int32)
  body_jntadr = np.full(nbody, -1, np.int32)
  body_dofnum = np.zeros(nbody, np.int32)
  body_dofadr = np.full(nbody, -1, np.int32)
  jnt_qposadr = np.zeros(njnt, np.int32)
  jnt_dofadr = np.zeros(njnt, np.int32)
  nq = nv = 0
  dof_body, dof_jnt = [], []
  qpos0, qpos_spring = [], []
  for j, jn in enumerate(c.joints):
    b = jn['body']
    if body_jntnum[b] == 0:
      body_jntadr[b] = j
      body_dofadr[b] = nv
    body_jntnum[b] += 1
    jnt_qposadr[j], jnt_dofadr[j] = nq, nv
    t = jn['type']
    nqj, nvj = {0: (7, 6), 1: (4, 3), 2: (1, 1), 3: (1, 1)}[t]
    if t == 0:
      bq = c.bodies[b]
      q0 = list(bq['pos']) + list(bq['quat'])
      qpos0 += q0
      qpos_spring += q0
    elif t == 1:
      qpos0 += [1, 0, 0, 0]
      qpos_spring += [1, 0, 0, 0]
    else:
      qpos0.append(jn['ref'])
      qpos_spring.append(jn['springref'])
    nq += nqj
    nv += nvj
    body_dofnum[b] += nvj
    dof_body += [b] * nvj
    dof_jnt += [j] * nvj
  # joints must be grouped by body in document order (they are: _body_children adds them before recursing)
  for b in range(nbody):
    if body_jntnum[b]:
      assert all(c.joints[body_jntadr[b] + k]['body'] == b for k in range(body_jntnum[b]))
  dof_body = np.array(dof_body, np.int32).reshape(-1)
  dof_jnt = np.array(dof_jnt, np.int32).reshape(-1)
  dof_parent = np.full(nv, -1, np.int32)
  for d in range(nv):
    b = dof_body[d]
    if d > body_dofadr[b]:
      dof_parent[d] = d - 1
    else:
      p = body_parent[b]
      while p > 0 and body_dofnum[p] == 0:
        p = body_parent[p]
      if p > 0:
        dof_parent[d] = body_dofadr[p] + body_dofnum[p] - 1
  body_root = np.zeros(nbody, np.int32)
  body_weld = np.zeros(nbody, np.int32)
  for b in range(1, nbody):
    p = body_parent[b]
    body_root[b] = b if p == 0 else body_root[p]
    body_weld[b] = b if body_jntnum[b] > 0 else body_weld[p]

  # ---- geoms grouped per body -------------------------------------------------------------
  order = sorted(range(ngeom), key=lambda g: (c.geoms[g]['body'], g))
  remap = {old: new for new, old in enumerate(order)}
  c.geoms = [c.geoms[g] for g in order]
  c.names['geom'] = {k: remap[v] for k, v in c.names['geom'].items()}
  sorder = sorted(range(nsite), key=lambda s: (c.sites[s]['body'], s))
  sremap = {old: new for new, old in enumerate(sorder)}
  c.sites = [c.sites[s] for s in sorder]
  c.names['site'] = {k: sremap[v] for k, v in c.names['site'].items()}
  body_geomnum = np.zeros(nbody, np.int32)
  body_geomadr = np.full(nbody, -1, np.int32)
  for g, gm in enumerate(c.geoms):
    b = gm['body']
    if body_geomnum[b] == 0:
      body_geomadr[b] = g
    body_geomnum[b] += 1

  # ---- inertial properties ----------------------------------------------------------------
  body_mass = np.zeros(nbody)
  body_ipos = np.zeros((nbody, 3))
  body_iquat = np.tile(np.array([1.0, 0, 0, 0]), (nbody, 1))
  body_inertia = np.zeros((nbody, 3))
  for b in range(1, nbody):
    bd = c.bodies[b]
    use_geoms = (c.inertiafromgeom == 'true') or (c.inertiafromgeom == 'auto' and bd['inertial'] is None)
    if not use_geoms:
      if bd['inertial'] is not None:
        it = bd['inertial']
        body_mass[b], body_ipos[b], body_iquat[b], body_inertia[b] = it['mass'], it['pos'], it['quat'], it['diag']
      continue
    gs = [g for g in c.geoms if g['body'] == b]
    masses, coms, tensors = [], [], []
    for g in gs:
      vol, unit_i = _geom_volume_inertia(g['type'], g['size'])
      m = g['mass'] if g['mass'] is not None else g['density'] * vol
      scale = (m / vol) if vol > 0 else 0.0
      R = quat_to_mat(g['quat'])
      masses.append(m)
      coms.append(g['pos'])
      tensors.append(R @ np.diag(unit_i * scale) @ R.T)
    mtot = float(sum(masses))
    if mtot <= 0:
      continue
    com = sum(m * p for m, p in zip(masses, coms)) / mtot
    full = np.zeros((3, 3))
    for m, p, T in zip(masses, coms, tensors):
      d = p - com
      full += T + m * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
    body_mass[b] = mtot
    body_ipos[b] = com
    live = [g for g, m in zip(gs, masses) if m > 0]
    if len(live) == 1:
      # single massive geom: its own frame is already principal
      g = live[0]
      _, unit_i = _geom_volume_inertia(g['type'], g['size'])
      vol = _geom_volume_inertia(g['type'], g['size'])[0]
      body_iquat[b] = g['quat']
      body_inertia[b] = unit_i * (mtot / vol)
    else:
      w, v = np.linalg.eigh(full)
      idx = np.argsort(-w)
      w, v = w[idx], v[:, idx]
      if np.linalg.det(v) < 0:
        v[:, 2] = -v[:, 2]
      body_iquat[b] = mat_to_quat(v)
      body_inertia[b] = w
  if c.boundmass > 0:
    body_mass[1:] = np.maximum(body_mass[1:], c.boundmass)
  if c.boundinertia > 0:
    body_inertia[1:] = np.maximum(body_inertia[1:], c.boundinertia)
  if c.settotalmass > 0:
    s = c.settotalmass / body_mass.sum()
    body_mass *= s
    body_inertia *= s
  subtree = body_mass.copy()
  for b in range(nbody - 1, 0, -1):
    subtree[body_parent[b]] += subtree[b]

  # ---- tree levels ------------------------------------------------------------------------
  depth = np.array([b['depth'] for b in c.bodies], np.int32)
  nlevel = int(depth.max()) + 1
  level_body = np.array(sorted(range(nbody), key=lambda b: (depth[b], b)), np.int32)
  level_adr = np.zeros(nlevel + 1, np.int32)
  for l in range(nlevel):
    level_adr[l + 1] = level_adr[l] + int((depth == l).sum())

  if nv > 64:
    raise NotImplementedError('models with more than 64 dofs are outside the supported subset')
  dofmask = np.zeros((nbody, 2), np.uint32)
  for b in range(1, nbody):
    p = body_parent[b]
    dofmask[b] = dofmask[p]
    for k in range(body_dofadr[b], body_dofadr[b] + body_dofnum[b]):
      dofmask[b, k // 32] |= np.uint32(1 << (k % 32))
  F['body_dofmask'] = dofmask.view(np.int32)
  F.update(body_parentid=body_parent, body_rootid=body_root, body_weldid=body_weld, body_jntnum=body_jntnum,
           body_jntadr=body_jntadr, body_dofnum=body_dofnum, body_dofadr=body_dofadr,
           body_geomnum=body_geomnum, body_geomadr=body_geomadr,
           body_pos=np.array([b['pos'] for b in c.bodies]), body_quat=np.array([b['quat'] for b in c.bodies]),
           body_ipos=body_ipos, body_iquat=body_iquat, body_mass=body_mass, body_subtreemass=subtree,
           body_inertia=body_inertia, level_adr=level_adr, level_body=level_body)

  J = c.joints
  F.update(jnt_type=np.array([j['type'] for j in J], np.int32), jnt_qposadr=jnt_qposadr, jnt_dofadr=jnt_dofadr,
           jnt_bodyid=np.array([j['body'] for j in J], np.int32),
           jnt_limited=np.array([j['limited'] for j in J], np.int32),
           jnt_pos=[j['pos'] for j in J], jnt_axis=[j['axis'] for j in J],
           jnt_stiffness=np.array([j['stiffness'] for j in J], np.float64),
           jnt_range=[j['range'] for j in J], jnt_margin=np.array([j['margin'] for j in J], np.float64),
           jnt_solref=[j['solref'] for j in J], jnt_solimp=[j['solimp'] for j in J],
           qpos0=np.array(qpos0, np.float64), qpos_spring=np.array(qpos_spring, np.float64))
  F.update(dof_bodyid=dof_body, dof_jntid=dof_jnt, dof_parentid=dof_parent,
           dof_armature=np.array([J[j]['armature'] for j in dof_jnt], np.float64),
           dof_damping=np.array([J[j]['damping'] for j in dof_jnt], np.float64),
           dof_frictionloss=np.array([J[j]['frictionloss'] for j in dof_jnt], np.float64),
           dof_solref=[J[j]['solreffriction'] for j in dof_jnt], dof_solimp=[J[j]['solimpfriction'] for j in dof_jnt])

  G = c.geoms
  F.update(geom_type=np.array([g['type'] for g in G], np.int32), geom_bodyid=np.array([g['body'] for g in G], np.int32),
           geom_condim=np.array([g['condim'] for g in G], np.int32),
           geom_contype=np.array([g['contype'] for g in G], np.int32),
           geom_conaffinity=np.array([g['conaffinity'] for g in G], np.int32),
           geom_priority=np.array([g['priority'] for g in G], np.int32),
           geom_size=[g['size'] for g in G], geom_pos=[g['pos'] for g in G], geom_quat=[g['quat'] for g in G],
           geom_rbound=np.array([_geom_rbound(g['type'], g['size']) for g in G], np.float64),
           geom_friction=[g['friction'] for g in G], geom_solmix=np.array([g['solmix'] for g in G], np.float64),
           geom_solref=[g['solref'] for g in G], geom_solimp=[g['solimp'] for g in G],
           geom_margin=np.array([g['margin'] for g in G], np.float64),
           geom_gap=np.array([g['gap'] for g in G], np.float64))
  S = c.sites
  F.update(site_bodyid=np.array([s['body'] for s in S], np.int32), site_type=np.array([s['type'] for s in S], np.int32),
           site_pos=[s['pos'] for s in S], site_quat=[s['quat'] for s in S], site_size=[s['size'] for s in S])

  # ---- contact candidate pairs (static filters applied once) -------------------------------
  excludes = set()
  contact = root.find('contact')
  if contact is not None:
    for ex in contact.findall('exclude'):
      b1, b2 = c.names['body'][ex.attrib['body1']], c.names['body'][ex.attrib['body2']]
      excludes.add((min(b1, b2), max(b1, b2)))
    if contact.findall('pair'):
      raise NotImplementedError('explicit <pair> contacts are outside the supported subset')
  filterparent = not (flags_dis & _DISABLE_BITS['filterparent'])
  pair1, pair2 = [], []
  for b1 in range(nbody):
    for b2 in range(b1 + 1, nbody):
      if body_geomnum[b1] == 0 or body_geomnum[b2] == 0:
        continue
      w1, w2 = body_weld[b1], body_weld[b2]
      if w1 == w2:
        continue
      if (b1, b2) in excludes:
        continue
      wp1 = body_weld[body_parent[w1]] if w1 else 0
      wp2 = body_weld[body_parent[w2]] if w2 else 0
      if filterparent and w1 != 0 and w2 != 0 and (w1 == wp2 or w2 == wp1):
        continue
      for g1 in range(body_geomadr[b1], body_geomadr[b1] + body_geomnum[b1]):
        for g2 in range(body_geomadr[b2], body_geomadr[b2] + body_geomnum[b2]):
          a, b = G[g1], G[g2]
          if not ((a['contype'] & b['conaffinity']) or (b['contype'] & a['conaffinity'])):
            continue
          if a['type'] == 0 and b['type'] == 0:
            continue
          if a['type'] > b['type']:
            pair1.append(g2)
            pair2.append(g1)
          else:
            pair1.append(g1)
            pair2.append(g2)
  F.update(pair_geom1=np.array(pair1, np.int32), pair_geom2=np.array(pair2, np.int32))

  # ---- tendons (fixed) --------------------------------------------------------------------
  tendons = []
  tnode = root.find('tendon')
  if tnode is not None:
    for t in tnode:
      if t.tag != 'fixed':
        raise NotImplementedError('spatial tendons are outside the supported subset')
      terms = [(c.names['joint'][jn.attrib['joint']], float(jn.attrib['coef'])) for jn in t.findall('joint')]
      name = t.attrib.get('name', f'_tendon{len(tendons)}')
      c.names['tendon'][name] = len(tendons)
      tendons.append(dict(name=name, terms=terms))
  ntendon = len(tendons)
  tendon_adr, tendon_num, wrap_objid, wrap_prm = [], [], [], []
  for t in tendons:
    tendon_adr.append(len(wrap_objid))
    tendon_num.append(len(t['terms']))
    for j, coef in t['terms']:
      if J[j]['type'] not in (2, 3):
        raise ValueError('fixed tendons couple scalar joints only')
      wrap_objid.append(j)
      wrap_prm.append(coef)
  q0 = np.array(qpos0, np.float64)
  tendon_length0 = np.array([sum(cf * q0[jnt_qposadr[j]] for j, cf in t['terms']) for t in tendons], np.float64)
  F.update(tendon_adr=np.array(tendon_adr, np.int32), tendon_num=np.array(tendon_num, np.int32),
           wrap_objid=np.array(wrap_objid, np.int32), wrap_prm=np.array(wrap_prm, np.float64),
           tendon_length0=tendon_length0)

  # ---- equality ---------------------------------------------------------------------------
  eqs = []
  enode = root.find('equality')
  if enode is not None:
    for e in enode:
      a = c.defaults.get('equality', e.attrib.get('class'))
      a.update(e.attrib)
      if e.tag == 'tendon':
        et = 3
        o1 = c.names['tendon'][a['tendon1']]
        o2 = c.names['tendon'][a['tendon2']] if 'tendon2' in a else -1
      elif e.tag == 'joint':
        et = 2
        o1 = c.names['joint'][a['joint1']]
        o2 = c.names['joint'][a['joint2']] if 'joint2' in a else -1
      else:
        raise NotImplementedError(f'<equality><{e.tag}> is outside the supported subset')
      data = np.zeros(11)
      data[:5] = _pad(_floats(a.get('polycoef', '0 1 0 0 0')), [0, 1, 0, 0, 0])
      name = a.get('name', f'_eq{len(eqs)}')
      c.names['equality'][name] = len(eqs)
      eqs.append(dict(type=et, o1=o1, o2=o2, active=a.get('active', 'true') == 'true', data=data,
                      solref=_floats(a.get('solref', '0.02 1'), 2), solimp=_solimp(a.get('solimp'))))
  F.update(eq_type=np.array([e['type'] for e in eqs], np.int32), eq_obj1id=np.array([e['o1'] for e in eqs], np.int32),
           eq_obj2id=np.array([e['o2'] for e in eqs], np.int32),
           eq_active0=np.array([e['active'] for e in eqs], np.int32), eq_data=[e['data'] for e in eqs],
           eq_solref=[e['solref'] for e in eqs], eq_solimp=[e['solimp'] for e in eqs])

  # ---- actuators --------------------------------------------------------------------------
  acts = []
  anode = root.find('actuator')
  if anode is not None:
    for e in anode:
      base = c.defaults.get('general', e.attrib.get('class'))
      if e.tag == 'general':
        a = dict(base)
        a.update(e.attrib)
      else:
        a = dict(base)
        a.update(_actuator_shortcut(e.tag, e.attrib, base))
      if 'joint' in a:
        trntype, trnid = 0, c.names['joint'][a['joint']]
        if J[trnid]['type'] not in (2, 3):
          raise NotImplementedError('actuators on ball/free joints are outside the supported subset')
      elif 'tendon' in a:
        trntype, trnid = 3, c.names['tendon'][a['tendon']]
      else:
        raise NotImplementedError('only joint and tendon transmissions are supported')
      dyntype = {'none': 0, 'integrator': 1, 'filter': 2, 'filterexact': 3}[a.get('dyntype', 'none')]
      if dyntype == 3:
        raise NotImplementedError('filterexact dynamics are outside the supported subset')
      gaintype = {'fixed': 0, 'affine': 1}[a.get('gaintype', 'fixed')]
      biastype = {'none': 0, 'affine': 1}[a.get('biastype', 'none')]
      ctrlrange = _floats(a.get('ctrlrange', '0 0'), 2)
      forcerange = _floats(a.get('forcerange', '0 0'), 2)
      actrange = _floats(a.get('actrange', '0 0'), 2)

      def lim(key, rng_key):
        v = a.get(key, 'auto')
        return (c.autolimits and rng_key in a) if v == 'auto' else v == 'true'
      name = a.get('name', f'_actuator{len(acts)}')
      c.names['actuator'][name] = len(acts)
      acts.append(dict(name=name, trntype=trntype, trnid=trnid, dyntype=dyntype, gaintype=gaintype,
                       biastype=biastype, gear=_pad(_floats(a.get('gear', '1')), [1, 0, 0, 0, 0, 0])[0],
                       gainprm=_pad(_floats(a.get('gainprm', '1')), [1, 0, 0]),
                       biasprm=_pad(_floats(a.get('biasprm', '0')), [0, 0, 0]),
                       dynprm=_pad(_floats(a.get('dynprm', '1')), [1, 0, 0])[0],
                       ctrllimited=lim('ctrllimited', 'ctrlrange'), forcelimited=lim('forcelimited', 'forcerange'),
                       actlimited=lim('actlimited', 'actrange'), ctrlrange=ctrlrange, forcerange=forcerange,
                       actrange=actrange))
  nu = len(acts)
  na = 0
  actadr = []
  for a in acts:
    if a['dyntype'] != 0:
      actadr.append(na)
      na += 1
    else:
      actadr.append(-1)
  F.update(actuator_trntype=np.array([a['trntype'] for a in acts], np.int32),
           actuator_trnid=np.array([a['trnid'] for a in acts], np.int32),
           actuator_dyntype=np.array([a['dyntype'] for a in acts], np.int32),
           actuator_gaintype=np.array([a['gaintype'] for a in acts], np.int32),
           actuator_biastype=np.array([a['biastype'] for a in acts], np.int32),
           actuator_ctrllimited=np.array([a['ctrllimited'] for a in acts], np.int32),
           actuator_forcelimited=np.array([a['forcelimited'] for a in acts], np.int32),
           actuator_actlimited=np.array([a['actlimited'] for a in acts], np.int32),
           actuator_actadr=np.array(actadr, np.int32),
           actuator_gear=np.array([a['gear'] for a in acts], np.float64),
           actuator_gainprm=[a['gainprm'] for a in acts], actuator_biasprm=[a['biasprm'] for a in acts],
           actuator_dynprm=np.array([a['dynprm'] for a in acts], np.float64),
           actuator_ctrlrange=[a['ctrlrange'] for a in acts], actuator_forcerange=[a['forcerange'] for a in acts],
           actuator_actrange=[a['actrange'] for a in acts])

  # ---- sensors ----------------------------------------------------------------------------
  sens = []
  snode = root.find('sensor')
  adr = 0
  if snode is not None:
    for e in snode:
      if e.tag not in _SENSOR_KINDS:
        raise NotImplementedError(f'sensor <{e.tag}> is outside the supported subset')
      stype, objtag, dim, stage = _SENSOR_KINDS[e.tag]
      a = e.attrib
      reftype, refid = 0, -1
      if e.tag == 'framepos':
        objtype = _OBJ[a['objtype']]
        key = 'body' if a['objtype'] in ('body', 'xbody') else a['objtype']
        objid = c.names[key][a['objname']]
        if 'reftype' in a:
          reftype = _OBJ[a['reftype']]
          rkey = 'body' if a['reftype'] in ('body', 'xbody') else a['reftype']
          refid = c.names[rkey][a['refname']]
      else:
        objtype = _OBJ[objtag]
        objid = c.names[objtag][a[objtag]]
      name = a.get('name', f'_sensor{len(sens)}')
      c.names['sensor'][name] = len(sens)
      sens.append(dict(name=name, type=stype, objtype=objtype, objid=objid, reftype=reftype, refid=refid, dim=dim,
                       adr=adr, stage=stage))
      adr += dim
  F.update(sensor_type=np.array([s['type'] for s in sens], np.int32),
           sensor_objtype=np.array([s['objtype'] for s in sens], np.int32),
           sensor_objid=np.array([s['objid'] for s in sens], np.int32),
           sensor_reftype=np.array([s['reftype'] for s in sens], np.int32),
           sensor_refid=np.array([s['refid'] for s in sens], np.int32),
           sensor_dim=np.array([s['dim'] for s in sens], np.int32), sensor_adr=np.array([s['adr'] for s in sens], np.int32),
           sensor_needstage=np.array([s['stage'] for s in sens], np.int32))

  # ---- keyframes --------------------------------------------------------------------------
  keys = []
  knode = root.find('keyframe')
  if knode is not None:
    for k in knode.findall('key'):
      kq = q0.copy()
      if 'qpos' in k.attrib:
        kq = _floats(k.attrib['qpos'], nq)
      c.names['key'][k.attrib.get('name', f'_key{len(keys)}')] = len(keys)
      keys.append(kq)
  F['key_qpos'] = keys

  # ---- sizes / capacities -----------------------------------------------------------------
  size_node = root.find('size')
  npair = len(pair1)
  if nconmax is None:
    # default per-env capacity: enough for every candidate pair to yield its maximum contact count
    nconmax = int(min(max(16, 2 * npair), 64)) if npair else 0
  # rows: equality + one limit row per limited scalar joint (at most one side active) + 4 per contact (pyramid)
  nlim = sum(1 for j in J if j['limited'])
  nfric = int(sum(1 for j in dof_jnt if J[j]['frictionloss'] > 0))
  if njmax is None:
    njmax = len(eqs) + nfric + nlim + 4 * nconmax
    njmax = int(min(njmax, 160))
  sizes = np.zeros(_model.NSIZES, np.int32)
  S_ = _model.SIZE
  for key, val in dict(NQ=nq, NV=nv, NU=nu, NA=na, NBODY=nbody, NJNT=njnt, NGEOM=ngeom, NSITE=nsite, NTENDON=ntendon,
                       NWRAP=len(wrap_objid), NEQ=len(eqs), NSENSOR=len(sens), NSENSORDATA=adr, NPAIR=npair,
                       NLEVEL=nlevel, NKEY=len(keys), NCONMAX=nconmax, NJMAX=njmax).items():
    sizes[S_[key]] = val
  F['sizes'] = sizes

  opt_real = np.zeros(_model.NOPTR)
  R_ = _model.OPTR
  opt_real[R_['TIMESTEP']] = timestep
  opt_real[R_['GRAVITY_X']:R_['GRAVITY_X'] + 3] = gravity
  opt_real[R_['TOLERANCE']] = float(opt.get('tolerance', 1e-8))
  opt_real[R_['LS_TOLERANCE']] = float(opt.get('ls_tolerance', 0.01))
  opt_real[R_['IMPRATIO']] = float(opt.get('impratio', 1))
  opt_int = np.zeros(_model.NOPTI, np.int32)
  I_ = _model.OPTI
  opt_int[I_['INTEGRATOR']] = integrator
  opt_int[I_['SOLVER']] = solver
  opt_int[I_['ITERATIONS']] = int(opt.get('iterations', 100))
  opt_int[I_['LS_ITERATIONS']] = int(opt.get('ls_iterations', 50))
  opt_int[I_['DISABLEFLAGS']] = flags_dis
  opt_int[I_['ENABLEFLAGS']] = flags_en
  opt_int[I_['CONE']] = cone

  # ---- mj_setConst equivalents (M^-1 at qpos0) ---------------------------------------------
  F['opt_real'], F['opt_int'] = opt_real, opt_int
  _set_const(F, nq, nv, nbody, tendons, jnt_qposadr, jnt_dofadr)

  names = {k: dict(v) for k, v in c.names.items()}
  names['model'] = {root.get('model', 'MuJoCo Model'): 0}
  extra = dict(light=c.lights, material=c.materials, texture=c.textures, numeric=c.custom['numeric'], text=c.custom['text'],
               tuple=c.custom['tuple'], equality=[e_['name'] for e_ in eqs] if eqs and isinstance(eqs[0], dict) and 'name' in eqs[0] else
               sorted(c.names.get('equality', {}), key=c.names.get('equality', {}).get))
  for k_, lst in extra.items():
    names[k_] = {n: i for i, n in enumerate(lst)}
  ordered = dict(body=[b['name'] for b in c.bodies], joint=[j['name'] for j in J], geom=[g['name'] for g in G],
                 site=[s['name'] for s in S], actuator=[a['name'] for a in acts],
                 tendon=[t['name'] for t in tendons], sensor=[s['name'] for s in sens],
                 camera=[cam['name'] for cam in c.cameras], **extra)
  return _model.Model(F, names, ordered, vis=_visual_tables(c, root, F, G, S))


def _visual_tables(c, root, F, G, S):
  """What a renderer needs and the physics does not: colours, visibility groups, cameras, the model's extent.

  Stands where mjModel's geom_rgba / geom_group / site_* / cam_* / vis.global / stat.{center,extent} stand in the
  reference (read by engine.py:642-946 through MuJoCo's mjv_updateScene); consumed by dm_control_b200/render.py."""
  glob = {}
  for v in root.findall('visual'):
    for g in v.findall('global'):
      glob.update(g.attrib)
  fovy0 = float(glob.get('fovy', 45))
  ncam = len(c.cameras)
  xpos0, xquat0, _, _ = _kin0(F, F['qpos0'])
  cam_pos0, cam_mat0 = np.zeros((ncam, 3)), np.zeros((ncam, 9))
  cam_poscom0 = np.zeros((ncam, 3))
  # subtree centres of mass at qpos0 (trackcom cameras keep their world offset from it)
  nbody = len(c.bodies)
  ipos0 = np.stack([xpos0[b] + rot_vec(xquat0[b], F['body_ipos'][b]) for b in range(nbody)]) if nbody else np.zeros((0, 3))
  msum = np.asarray(F['body_mass'], dtype=np.float64).copy()
  mpos = ipos0 * msum[:, None]
  for b in range(nbody - 1, 0, -1):
    p = F['body_parentid'][b]
    msum[p] += msum[b]; mpos[p] += mpos[b]
  scom0 = np.where(msum[:, None] > 0, mpos / np.maximum(msum[:, None], 1e-300), xpos0)
  for k, cam in enumerate(c.cameras):
    b = cam['body']
    cam_pos0[k] = xpos0[b] + rot_vec(xquat0[b], cam['pos'])
    cam_mat0[k] = quat_to_mat(quat_mul(xquat0[b], cam['quat'])).reshape(-1)
    cam_poscom0[k] = cam_pos0[k] - scom0[b]
  # extent / centre from the geoms' bounding spheres at qpos0 (MuJoCo: mj_setConst -> stat.center, stat.extent)
  if G:
    gp = np.stack([xpos0[g['body']] + rot_vec(xquat0[g['body']], g['pos']) for g in G])
    rb = np.array([0.0 if g['type'] == 0 else _geom_rbound(g['type'], g['size']) for g in G])
    lo, hi = (gp - rb[:, None]).min(0), (gp + rb[:, None]).max(0)
    center = 0.5 * (lo + hi)
    extent = float(max(0.5 * np.linalg.norm(hi - lo), 1e-5))
  else:
    center, extent = np.zeros(3), 1.0
  stat = {}
  for st in root.findall('statistic'):
    stat.update(st.attrib)
  if 'extent' in stat:
    extent = float(stat['extent'])
  if 'center' in stat:
    center = _floats(stat['center'], 3)
  return dict(
      geom_rgba=np.array([g['rgba'] for g in G], dtype=np.float32).reshape(-1, 4),
      geom_group=np.array([g['group'] for g in G], dtype=np.int32),
      site_rgba=np.array([s_['rgba'] for s_ in S], dtype=np.float32).reshape(-1, 4),
      site_group=np.array([s_['group'] for s_ in S], dtype=np.int32),
      cam_bodyid=np.array([cam['body'] for cam in c.cameras], dtype=np.int32),
      cam_mode=np.array([cam['mode'] for cam in c.cameras], dtype=np.int32),
      cam_targetbodyid=np.array([c.names['body'].get(cam['target'], -1) if cam['target'] else -1 for cam in c.cameras], dtype=np.int32),
      cam_pos=np.array([cam['pos'] for cam in c.cameras], dtype=np.float64).reshape(-1, 3),
      cam_quat=np.array([cam['quat'] for cam in c.cameras], dtype=np.float64).reshape(-1, 4),
      cam_fovy=np.array([cam['fovy'] if cam['fovy'] is not None else fovy0 for cam in c.cameras], dtype=np.float64),
      cam_pos0=cam_pos0 - (xpos0[[cam['body'] for cam in c.cameras]] if ncam else np.zeros((0, 3))),
      cam_poscom0=cam_poscom0, cam_mat0=cam_mat0,
      mat_rgba=np.array([c.material_rgba[n] for n in c.materials], dtype=np.float32).reshape(-1, 4),
      global_fovy=np.array([fovy0]), stat_center=np.asarray(center, dtype=np.float64), stat_extent=np.array([extent]))


# ---------------------------------------------------------------------------------------------
# qpos0 statics: kinematics, joint-space inertia, Jacobians (numpy, compile time only)
# ---------------------------------------------------------------------------------------------

def _kin0(F, qpos):
  nbody = F['body_parentid'].shape[0]
  xpos = np.zeros((nbody, 3))
  xquat = np.tile(np.array([1.0, 0, 0, 0]), (nbody, 1))
  njnt = F['jnt_type'].shape[0]
  xanchor = np.zeros((njnt, 3))
  xaxis = np.zeros((njnt, 3))
  for b in range(1, nbody):
    p = F['body_parentid'][b]
    pos = xpos[p] + rot_vec(xquat[p], F['body_pos'][b])
    quat = quat_mul(xquat[p], F['body_quat'][b])
    for j in range(F['body_jntadr'][b], F['body_jntadr'][b] + F['body_jntnum'][b]):
      t, qa = F['jnt_type'][j], F['jnt_qposadr'][j]
      if t == 0:
        pos = qpos[qa:qa + 3].copy()
        quat = qpos[qa + 3:qa + 7] / np.linalg.norm(qpos[qa + 3:qa + 7])
        xanchor[j], xaxis[j] = pos, rot_vec(quat, F['jnt_axis'][j])
        continue
      xanchor[j] = pos + rot_vec(quat, F['jnt_pos'][j])
      xaxis[j] = rot_vec(quat, F['jnt_axis'][j])
      if t == 2:
        pos = pos + xaxis[j] * (qpos[qa] - F['qpos0'][qa])
      elif t == 3:
        quat = quat_mul(quat, axisangle_to_quat(F['jnt_axis'][j], qpos[qa] - F['qpos0'][qa]))
        pos = xanchor[j] - rot_vec(quat, F['jnt_pos'][j])
      else:
        quat = quat_mul(quat, qpos[qa:qa + 4] / np.linalg.norm(qpos[qa:qa + 4]))
        pos = xanchor[j] - rot_vec(quat, F['jnt_pos'][j])
    xpos[b], xquat[b] = pos, quat / np.linalg.norm(quat)
  return xpos, xquat, xanchor, xaxis


def _body_jac(F, xpos, xquat, xanchor, xaxis, body, point, nv):
  """Translational and rotational Jacobian (3 x nv each) of `point` attached to `body`."""
  jp, jr = np.zeros((3, nv)), np.zeros((3, nv))
  b = body
  while b > 0:
    for j in range(F['body_jntadr'][b], F['body_jntadr'][b] + F['body_jntnum'][b]):
      t, d = F['jnt_type'][j], F['jnt_dofadr'][j]
      if t == 0:
        jp[:, d:d + 3] = np.eye(3)
        R = quat_to_mat(xquat[b])
        for k in range(3):
          jr[:, d + 3 + k] = R[:, k]
          jp[:, d + 3 + k] = np.cross(R[:, k], point - xpos[b])
      elif t == 1:
        R = quat_to_mat(xquat[b])
        for k in range(3):
          jr[:, d + k] = R[:, k]
          jp[:, d + k] = np.cross(R[:, k], point - xanchor[j])
      elif t == 2:
        jp[:, d] = xaxis[j]
      else:
        jr[:, d] = xaxis[j]
        jp[:, d] = np.cross(xaxis[j], point - xanchor[j])
    b = F['body_parentid'][b]
  return jp, jr


def _set_const(F, nq, nv, nbody, tendons, jnt_qposadr, jnt_dofadr):
  q0 = F['qpos0']
  xpos, xquat, xanchor, xaxis = _kin0(F, q0)
  M = np.zeros((nv, nv))
  xipos = np.zeros((nbody, 3))
  for b in range(1, nbody):
    R = quat_to_mat(xquat[b])
    xipos[b] = xpos[b] + R @ F['body_ipos'][b]
    if F['body_mass'][b] <= 0 and not np.any(F['body_inertia'][b] > 0):
      continue
    Ri = quat_to_mat(quat_mul(xquat[b], F['body_iquat'][b]))
    Iw = Ri @ np.diag(F['body_inertia'][b]) @ Ri.T
    jp, jr = _body_jac(F, xpos, xquat, xanchor, xaxis, b, xipos[b], nv)
    M += F['body_mass'][b] * jp.T @ jp + jr.T @ Iw @ jr
  M += np.diag(F['dof_armature'])
  F['opt_real'][_model.OPTR['MEANINERTIA']] = float(np.mean(np.diag(M))) if nv else 1.0
  try:
    Minv = np.linalg.inv(M) if nv else np.zeros((0, 0))
  except np.linalg.LinAlgError:
    # a singular inertia matrix at qpos0 (e.g. several hinges about one axis on one body, as in the reference's
    # randomizers_test.py:76-86): MuJoCo still compiles such a model; the inverse weights come from the pseudo-inverse
    Minv = np.linalg.pinv(M)
  dof_inv = np.zeros(nv)
  for j in range(F['jnt_type'].shape[0]):
    t, d = F['jnt_type'][j], jnt_dofadr[j]
    if t == 0:
      dof_inv[d:d + 3] = np.mean(np.diag(Minv)[d:d + 3])
      dof_inv[d + 3:d + 6] = np.mean(np.diag(Minv)[d + 3:d + 6])
    elif t == 1:
      dof_inv[d:d + 3] = np.mean(np.diag(Minv)[d:d + 3])
    else:
      dof_inv[d] = Minv[d, d]
  F['dof_invweight0'] = dof_inv
  binv = np.zeros((nbody, 2))
  for b in range(1, nbody):
    if F['body_weldid'][b] == 0 or nv == 0:
      continue
    jp, jr = _body_jac(F, xpos, xquat, xanchor, xaxis, b, xipos[b], nv)
    binv[b, 0] = max(np.trace(jp @ Minv @ jp.T) / 3.0, 1e-15)
    binv[b, 1] = max(np.trace(jr @ Minv @ jr.T) / 3.0, 1e-15)
  F['body_invweight0'] = binv
  tinv = np.zeros(len(tendons))
  for i, t in enumerate(tendons):
    jt = np.zeros(nv)
    for j, cf in t['terms']:
      jt[jnt_dofadr[j]] += cf
    tinv[i] = jt @ Minv @ jt
  F['tendon_invweight0'] = tinv
