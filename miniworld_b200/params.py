"""Domain-randomisation parameter table (host side).

Mirrors the interface of the reference's `miniworld/params.py` (DomainParams.set /
get_max / sample / sample_many / no_random / copy and the DEFAULT_PARAMS table,
reference params.py:85-130) so level definitions written against the reference run
unchanged.  Sampling semantics that the device reset kernel reproduces
(csrc/reset.cuh): `rng is None` -> default value, float -> `rng.uniform(min, max)`
(element order for vectors), int -> `rng.integers(min, max + 1)`.
"""
import copy as _copy
from typing import NamedTuple

import numpy as np


class DomainParam(NamedTuple):
    default: object
    min: object
    max: object
    type: str


class DomainParams:
    DomainParam = DomainParam

    def __init__(self):
        self.params = {}

    def copy(self):
        return _copy.deepcopy(self)

    def no_random(self):
        """Copy whose ranges are collapsed onto the defaults (randomisation off)."""
        frozen = self.copy()
        frozen.params = {k: DomainParam(p.default, p.default, p.default, p.type)
                         for k, p in frozen.params.items()}
        return frozen

    def set(self, name, default, min=None, max=None, type="float"):
        default, min, max = (np.array(v) if isinstance(v, list) else v for v in (default, min, max))
        min = default if min is None else min
        max = default if max is None else max
        if isinstance(default, np.ndarray):
            if not (max.shape == default.shape == min.shape):
                raise AssertionError("shape mismatch for parameter %r" % name)
            if not (np.all(max >= default) and np.all(default >= min)):
                raise AssertionError("range must bracket the default for %r" % name)
            if type == "float":
                default, min, max = (v.astype("float") for v in (default, min, max))
        elif not (max >= default >= min):
            raise AssertionError("range must bracket the default for %r" % name)
        old = self.params.get(name)
        if old is not None:
            assert old.type == type
            if isinstance(old.default, np.ndarray):
                assert default.shape == old.default.shape
        self.params[name] = DomainParam(default, min, max, type)

    def get_max(self, name):
        return self.params[name].max

    def sample(self, rng, name):
        p = self.params[name]
        if rng is None:
            return p.default
        if p.type == "float":
            return rng.uniform(p.min, p.max)
        if p.type == "int":
            return rng.integers(p.min, p.max + 1)
        raise AssertionError("unknown parameter type %r" % p.type)

    def sample_many(self, rng, target_obj, param_names):
        for name in param_names:
            setattr(target_obj, name, self.sample(rng, name))


def _defaults():
    t = DomainParams()
    rows = [
        ("sky_color", [0.25, 0.82, 1], [0.1, 0.1, 0.1], [1.0, 1.0, 1.0]),
        ("light_pos", [0, 2.5, 0], [-40, 2.5, -40], [40, 5, 40]),
        ("light_color", [0.7, 0.7, 0.7], [0.45, 0.45, 0.45], [0.8, 0.8, 0.8]),
        ("light_ambient", [0.45, 0.45, 0.45], [0.35, 0.35, 0.35], [0.55, 0.55, 0.55]),
        ("obj_color_bias", [0, 0, 0], [-0.2, -0.2, -0.2], [0.2, 0.2, 0.2]),
        ("forward_step", 0.15, 0.12, 0.17),
        ("forward_drift", 0, -0.05, 0.05),
        ("turn_step", 15, 10, 20),
        ("bot_radius", 0.4, 0.38, 0.42),
        ("cam_pitch", 0, -5, 5),
        ("cam_fov_y", 60, 55, 65),
        ("cam_height", 1.5, 1.45, 1.55),
        ("cam_fwd_disp", 0, -0.05, 0.10),
    ]
    for row in rows:
        t.set(*row)
    return t


DEFAULT_PARAMS = _defaults()


def overlay_params(params, design):
    """A copy of `params` overlaid by `design` {name: (default, min, max)}, element by element as an env params row of
    the batched engine overlays its level's: a finite default replaces the param's, a finite (min, max) pair its range;
    None or NaN entries keep the param's.  The result is built without DomainParams.set's checks, so a range may lie
    outside its default or have min > max (numpy's uniform() takes both)."""
    out = params.copy()
    for name, row in design.items():
        p = out.params[name]
        if p.type != "float":
            raise TypeError("%r is a %s param; only float params can be designed" % (name, p.type))
        shape = np.shape(p.default)
        d, lo, hi = (np.full(shape, np.nan) if v is None else np.broadcast_to(np.asarray(v, np.float64), shape)
                     for v in row)
        rng = np.isfinite(lo) & np.isfinite(hi)
        vals = [np.where(np.isfinite(d), d, p.default), np.where(rng, lo, p.min), np.where(rng, hi, p.max)]
        vals = [np.array(v, np.float64) if shape else float(v) for v in vals]
        out.params[name] = DomainParam(vals[0], vals[1], vals[2], p.type)
    return out
