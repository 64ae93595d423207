"""Host-side mirror of the reference's ``FieldSet`` / ``Field`` / ``VectorField`` / ``XGrid``
for the hot path: it only *describes* the arrays; the velocity data itself is pinned in HBM by
the engine the first time a ParticleSet executes on it (reference: ``_core/fieldset.py``,
``_core/field.py``, ``_core/xgrid.py``, ``_core/model.py``).
"""

from __future__ import annotations

import warnings

import numpy as np

from .engine import Engine

EARTH_RADIUS = 6366707.019493707  # reference _core/mesh.py:6

__all__ = ["Field", "FieldSet", "VectorField", "XGrid"]


def window_range(time_s, t, sign: int, window: int) -> tuple[int, int]:
    """Time levels [first, first + n) to keep resident so that a particle at time ``t`` can step in direction
    ``sign`` (reference analogue: the span a WindowedArray keeps, _core/_windowed_array.py:56-97)."""
    T = len(time_s)
    if sign > 0:
        first = int(np.clip(np.searchsorted(time_s, t, side="right") - 1, 0, max(T - 2, 0)))
    else:
        last = int(np.clip(np.searchsorted(time_s, t, side="left"), 1, T - 1))
        first = max(0, last - window + 1)
    first = min(first, max(T - window, 0))
    return first, min(window, T - first)


def window_span(time_s, lo, hi, sign: int, window: int) -> tuple[int, int] | None:
    """Time levels [first, first + n) to keep resident so that every sample time in [lo, hi] (inside the time axis) reads
    resident levels; the window extends in direction ``sign`` beyond the span.  None when the span needs more than ``window``
    levels."""
    T = len(time_s)
    first = int(np.clip(np.searchsorted(time_s, lo, side="right") - 1, 0, max(T - 2, 0)))
    last = int(np.clip(np.searchsorted(time_s, hi, side="left"), 1, T - 1))
    if last - first + 1 > window:
        return None
    if sign < 0:
        first = max(0, last - window + 1)
    first = min(first, max(T - window, 0))
    return first, min(window, T - first)


def _to_seconds(time):
    """time axis -> (float64 seconds since the first level, origin) (reference index_search.py:88)."""
    if time is None:
        return None, None
    time = np.asarray(time)
    if time.size < 2:  # a single level is "no time dimension" (model.py:511-515)
        return None, None
    if np.issubdtype(time.dtype, np.datetime64) or np.issubdtype(time.dtype, np.timedelta64):
        sec = ((time - time[0]) / np.timedelta64(1, "s")).astype(np.float64)
        return sec, time[0]
    sec = time.astype(np.float64)
    return sec - sec[0], sec[0]


def _is_device_array(a) -> bool:
    """An array that already lives in HBM (torch CUDA tensor, CuPy array ...): exposes __cuda_array_interface__."""
    try:
        return isinstance(a.__cuda_array_interface__, dict)
    except Exception:  # absent, or a torch CPU tensor (the property raises)
        return False


def _batch_skips_hint(grid, hint) -> bool:
    """Curvilinear grids: the reference tests the hinted cells only `if np.any(xi)` (_core/index_search.py:269) -- when the hinted
    xi of EVERY sample is 0 (a fresh ParticleSet) the whole batch goes straight to the spatial hash."""
    return bool(grid.curvilinear and hint is not None and not np.any((np.asarray(hint).astype(np.int64) % grid.xdim) != 0))


class SphericalMesh:
    """``mesh=SphericalMesh(radius=...)`` (reference _core/mesh.py:23-51): a spherical mesh with a configurable planetary radius in
    metres (default: the Earth's, for which a degree of arc is exactly 1852 * 60 m)."""

    def __init__(self, radius=EARTH_RADIUS):
        if not isinstance(radius, (int, float, np.number)) or isinstance(radius, bool):
            raise TypeError(f"radius must be a number, got {type(radius).__name__}")
        if radius <= 0:
            raise ValueError(f"radius must be positive, got {radius}")
        self.radius = radius

    deg2m = property(lambda self: self.radius * np.pi / 180.0)

    def is_spherical(self):
        return True

    def __eq__(self, other):
        return isinstance(other, SphericalMesh) and self.radius == other.radius

    def __hash__(self):
        return hash((True, self.radius))

    def __repr__(self):
        return f"SphericalMesh(radius={self.radius!r})"


class XGrid:
    """Structured grid (rectilinear: 1-D lon/lat; depth optional).  ``xdim/ydim/zdim`` are cell
    counts as in the reference (``_core/xgrid.py:21-24,208-231``); they default to nodes - 1,
    which is what LOW/HIGH SGRID padding gives."""

    def __init__(self, lon, lat, depth=None, mesh="spherical", radius=None, xdim=None, ydim=None, zdim=None):
        self.lon = np.asarray(lon)
        self.lat = np.asarray(lat)
        self.depth = None if depth is None else np.asarray(depth)
        if self.lon.ndim not in (1, 2) or self.lat.ndim != self.lon.ndim:
            raise ValueError("lon/lat must both be 1-D (rectilinear) or both 2-D (curvilinear, shape (ny, nx))")
        if self.lon.ndim == 2 and self.lon.shape != self.lat.shape:
            raise ValueError("curvilinear lon and lat must share one shape (ny, nx)")
        if isinstance(mesh, SphericalMesh):  # reference: mesh=SphericalMesh(radius=...)
            mesh, radius = "spherical", (mesh.radius if radius is None else radius)
        if mesh not in ("flat", "spherical"):
            raise ValueError(f"mesh must be 'flat', 'spherical' or a SphericalMesh. Got {mesh!r}")
        self.mesh = mesh
        self.radius = (EARTH_RADIUS if radius is None else radius) if mesh == "spherical" else None
        self.xdim = self.lon.shape[-1] - 1 if xdim is None else xdim
        self.ydim = self.lat.shape[0] - 1 if ydim is None else ydim
        self._hash = None
        self.zdim = None if self.depth is None else (self.depth.size - 1 if zdim is None else zdim)

    @property
    def curvilinear(self):
        return self.lon.ndim == 2

    def get_spatial_hash(self, table=False):
        """reference _core/basegrid.py:192-216: built lazily, once.  ``table=False``: only the per-face quantised boxes
        (the float part); the engine expands / sorts / compresses them into the table on the device."""
        if self._hash is None or (table and "keys" not in self._hash):
            from .spatialhash import build_spatial_hash

            self._hash = build_spatial_hash(self.lon, self.lat, self.is_spherical(), table=table)
        return self._hash

    def is_spherical(self):
        return self.mesh == "spherical"

    @property
    def deg2m(self):  # reference _core/xgrid.py:201-206, _core/mesh.py:37-40
        return self.radius * np.pi / 180.0 if self.mesh == "spherical" else 1.0

    @property
    def axes(self):
        return (["Z"] if self.depth is not None else []) + ["Y", "X"]


class Field:
    """Scalar field on the fieldset's grid (reference ``_core/field.py:46-202``).  ``interp_method``: "linear" (XLinear),
    "nearest" (XNearest), "cgrid_tracer" (CGrid_Tracer) or "constant" (XConstantField, a 1-node grid)."""

    def __init__(self, name, data, grid, fieldset, interp_method="linear", slot=None, host=None, windowed=False):
        self.name = name
        self.data = data
        self.grid = grid
        self._fieldset = fieldset
        self._host = host  # who keeps this field's grid in HBM: the FieldSet (None) or an _ExtraGrid of it
        self.interp_method = interp_method
        self._slot = slot  # device field slot (include/parcels_b200.h: 0..2 = U, V, W; 3.. = scalar fields)
        self._windowed = windowed  # only the host's time window of `data`'s levels is in HBM (time-slab streaming)

    def eval(self, t, z, y, x, particles=None, *, device=None, positions_are_f32=None):
        """``fieldset.P.eval(t, z, y, x[, particles])`` (reference _core/field.py:144-191), evaluated ON THE DEVICE
        (``pb_sample_scalar``); out-of-bounds samples are 0.  With ``particles`` the search is hinted by, and writes
        back, ``particles.ei[:, -1]`` and raises ``particles.state`` like the reference."""
        from .statuscodes import StatusCode

        fs = self._fieldset
        z, y, x = (np.atleast_1d(a.__array__() if hasattr(a, "__array__") else a) for a in (z, y, x))
        if self.interp_method == "constant":
            # XConstantField on its 1-node grid (_xinterpolators.py:156-166, model.py:292-318): index 0 everywhere
            if particles is not None:
                particles.ei[:, -1] = 0
            return float(np.asarray(self.data)[0, 0, 0, 0]) * np.ones_like(x)
        if self._slot is None:
            raise NotImplementedError(f"field {self.name!r} is not a sampled field of this FieldSet")
        if self.name in ("U", "V", "W"):
            warnings.warn("Sampling of velocities should normally be done using fieldset.UV or fieldset.UVW object; tread carefully",
                          RuntimeWarning, stacklevel=2)  # fmt: skip
        if device is None:
            device = next(iter(fs._engines), 0)
        t = np.atleast_1d(t.__array__() if hasattr(t, "__array__") else t)
        if np.issubdtype(t.dtype, np.floating) and np.any(np.isnan(t)):
            raise ValueError(f"Time values for particles with indices {np.where(np.isnan(t))[0]} cannot be NaN.")
        if positions_are_f32 is None:
            positions_are_f32 = all(a.dtype == np.float32 for a in (z, y, x))
        # the reference hints EVERY field's search with the last `ei` column, whatever the field's grid (`igrid` stays -1,
        # _core/field.py:101,173) and writes that field's cell back into it
        hint = None if particles is None else np.ascontiguousarray(np.asarray(particles.ei)[:, -1])
        host = self._host or fs
        if _batch_skips_hint(self.grid, hint):
            hint = None
        eng = host.engine(device)
        if self._windowed:
            host.cover_window(device, t)  # the batch's levels resident (times outside the axis: OutsideTimeInterval)
        val, ei, st = eng.sample_scalar(self._slot, self.interp_method, t, z, y, x, positions_are_f32=positions_are_f32,
                                        ei_hint=hint)  # fmt: skip
        if particles is not None:
            particles.ei[:, -1] = ei
            state = np.asarray(particles.state)
            if np.any(st == StatusCode.ErrorOutsideTimeInterval):  # whole view flagged, 0 returned (field.py:31-44)
                particles.state = StatusCode.ErrorOutsideTimeInterval
                val[:] = 0
            else:
                particles.state = np.where(st >= StatusCode.Error, np.maximum(state, st), state)
        return val.reshape(np.shape(x))

    def __getitem__(self, key):
        if hasattr(key, "_data") and not isinstance(key, tuple):  # a ParticleSet / ParticleSetView
            return self.eval(key.t, key.z, key.y, key.x, key)
        return self.eval(*key)


class VectorField:
    def __init__(self, name, U, V, W=None, host=None):
        self.name, self.U, self.V, self.W = name, U, V, W
        self.grid = U.grid
        self.vector_type = "3D" if W is not None else "2D"
        self._host = host  # who keeps the components in HBM: the FieldSet (None) or an _ExtraGrid (a vector field on another grid)

    def eval(self, t, z, y, x, particles=None, *, device=None, positions_are_f32=None):
        """``fieldset.UV.eval(t, z, y, x[, particles])`` (reference _core/field.py:250-295), evaluated ON THE DEVICE
        (``pb_sample_velocity``).  Returns (u, v) or (u, v, w) float64 arrays; out-of-bounds samples are 0.  With
        ``particles`` (a ParticleSet or the ParticleSetView a user kernel received) the search is hinted by, and
        writes back, ``particles.ei[:, -1]`` and raises ``particles.state`` exactly like the reference does."""
        fs = self.U._fieldset
        host = self._host or fs
        if device is None:
            device = next(iter(fs._engines), 0)
        z, y, x = (np.atleast_1d(a.__array__() if hasattr(a, "__array__") else a) for a in (z, y, x))
        t = np.atleast_1d(t.__array__() if hasattr(t, "__array__") else t)
        if np.issubdtype(t.dtype, np.floating) and np.any(np.isnan(t)):  # reference _core/field.py:396-398
            raise ValueError(f"Time values for particles with indices {np.where(np.isnan(t))[0]} cannot be NaN.")
        if positions_are_f32 is None:
            positions_are_f32 = all(a.dtype == np.float32 for a in (z, y, x))
        hint = None
        if particles is not None:
            hint = np.ascontiguousarray(np.asarray(particles.ei)[:, -1])
        eng = host.engine(device)
        if self.U._windowed:
            host.cover_window(device, t)  # time-windowed U, V, W: the batch's levels resident (times outside the axis: OutsideTimeInterval)
        u, v, w, ei, st = eng.sample_velocity(t, z, y, x, three_d=self.W is not None, positions_are_f32=positions_are_f32,
                                                              ei_hint=hint, no_hint=_batch_skips_hint(self.grid, hint))  # fmt: skip
        if particles is not None:
            from .statuscodes import StatusCode

            particles.ei[:, -1] = ei
            state = np.asarray(particles.state)
            if np.any(st == StatusCode.ErrorOutsideTimeInterval):  # whole view flagged, zeros returned (field.py:31-44)
                particles.state = StatusCode.ErrorOutsideTimeInterval
                u[:] = 0
                v[:] = 0
                w[:] = 0
            else:
                particles.state = np.where(st >= StatusCode.Error, np.maximum(state, st), state)
        shape = np.shape(x)
        return (u.reshape(shape), v.reshape(shape)) + ((w.reshape(shape),) if self.W is not None else ())

    def __getitem__(self, key):
        if hasattr(key, "_data") and not isinstance(key, tuple):  # a ParticleSet / ParticleSetView
            return self.eval(key.t, key.z, key.y, key.x, key)
        return self.eval(*key)


def _field_data(name, data, time_window):
    """The data of a scalar field: a float32 / float64 (T, Z, Y, X) array uploaded whole, or with ``time_window`` the caller's
    array-like (np.memmap, a lazy loader ...) itself, of which only ``data[level]`` is ever read."""
    if time_window is None:
        data = np.ascontiguousarray(data)
        if data.ndim != 4:
            raise ValueError(f"{name} must be laid out (T, Z, Y, X); got shape {data.shape}")
        return data if data.dtype in (np.float32, np.float64) else data.astype(np.float64)
    shape = tuple(data.shape)
    if len(shape) != 4:
        raise ValueError(f"{name} must be laid out (T, Z, Y, X); got shape {shape}")
    if np.dtype(data.dtype) not in (np.float32, np.float64):
        raise ValueError(f"{name}: a time-windowed field must be float32 or float64, got {data.dtype}")
    if shape[0] < 2:
        raise ValueError(f"{name} has a single time level: there is no time dimension to stream (add it without time_window)")
    return data


class _TimeWindow:
    """Time-slab streaming of the windowed fields of one device engine per device (the FieldSet's velocity grid, or an
    _ExtraGrid): ``time_window`` consecutive levels of the time axis ``_time_s`` resident, plus one ring slot that receives the
    next level.  The owner has ``_engines``, ``_win`` (device -> window state) and ``_windowed_fields()`` -> [(slot, data)]."""

    def _load_level(self, eng, device, level):
        w = self._win[device]
        ring = self.time_window + 1
        w["resident"] = {lv for lv in w["resident"] if lv % ring != level % ring}
        for slot, data in self._windowed_fields():
            eng.window_load(slot, level, np.asarray(data[level]))
        w["resident"].add(level)

    def _window_add_field(self, slot, data):
        """A windowed field added after the engines were made: its ring on each, holding the levels resident there."""
        for device, eng in self._engines.items():
            eng.window_create(slot, data.dtype, data.shape, self.time_window)
            w = self._win[device]
            for lv in sorted(w["resident"]):
                eng.window_load(slot, lv, np.asarray(data[lv]))
            if w["n"]:
                eng.window_set(w["first"], w["n"])

    def slide_window(self, device, t, sign):
        """Make the levels a particle at time ``t`` needs resident; returns True if the window moved."""
        return self._set_window(device, *window_range(self._time_s, t, sign, self.time_window))

    def cover_window(self, device, t, sign=1):
        """Make the levels of every finite sample time in ``t`` that lies inside the time axis resident (a step-by-step kernel
        list, a user kernel's ``fieldset.UV[...]``).  Raises RuntimeError when no window of ``time_window`` levels holds them."""
        t = np.asarray(t, dtype=np.float64)
        inside = t[(t >= self._time_s[0]) & (t <= self._time_s[-1])]  # (NaN fails both tests)
        if inside.size == 0:
            return
        lo, hi = float(inside.min()), float(inside.max())
        w = self._win[device]
        if w["n"] and self._time_s[w["first"]] <= lo and hi <= self._time_s[w["first"] + w["n"] - 1]:
            return
        span = window_span(self._time_s, lo, hi, sign, self.time_window)
        if span is None:
            raise RuntimeError(f"sample times {lo} .. {hi} span more than the {self.time_window} resident time levels of this "
                               "FieldSet: widen time_window")  # fmt: skip
        self._set_window(device, *span)

    def _set_window(self, device, first, n):
        eng = self._engines[device]
        w = self._win[device]
        moved = (first, n) != (w["first"], w["n"])
        for lv in range(first, first + n):
            if lv not in w["resident"]:
                self._load_level(eng, device, lv)
        eng.window_set(first, n)
        w["first"], w["n"] = first, n
        return moved

    def prefetch_next(self, device, sign):
        """Start copying the level the next window will need into the spare ring slot (overlaps the kernel)."""
        w = self._win[device]
        nxt = w["first"] + w["n"] if sign > 0 else w["first"] - 1
        if 0 <= nxt < len(self._time_s) and nxt not in w["resident"]:
            self._load_level(self._engines[device], device, nxt)


class _ExtraGrid(_TimeWindow):
    """A further XGrid of the FieldSet (reference: every Field carries its own grid, _core/field.py:102-134; the gridset is the
    list of distinct grids, _core/fieldset.py:225-235) with the scalar fields that live on it.  Each grid is resident in its own
    device engine (grid axes / spatial hash + field slots 3..15); the advection kernels only ever see the velocity grid.
    Fields added with ``time_window=W`` stream through one window of W levels over this grid's time axis, slid by the
    ``eval`` of its fields."""

    def __init__(self, grid, time_s):
        self.grid, self._time_s = grid, time_s
        self.fields = []
        self.vector = None  # (U, V, W or None) Field objects of a vector field on this grid: device slots 0..2
        self.vector_interp, self.offsets = None, (1, 1, 0)
        self.time_window = None  # levels resident of the windowed fields (one window for all of them)
        self._engines = {}
        self._win = {}

    def _windowed_fields(self):
        return [(f._slot, f.data) for f in (*(self.vector or ()), *self.fields) if f is not None and f._windowed]

    def use_window(self, name, time_window):
        """Check ``time_window=`` of a field added to this grid: one window for every windowed field of the grid."""
        if self._time_s is None:
            raise ValueError(f"{name}: time_window on a grid without a time axis (no time dimension to stream)")
        time_window = int(time_window)
        if self.time_window is not None and time_window != self.time_window:
            raise ValueError(f"{name}: time_window={time_window}, but the windowed fields of its grid use {self.time_window}")
        self.time_window = time_window

    def engine(self, device: int = 0) -> Engine:
        eng = self._engines.get(device)
        if eng is None:
            eng = Engine(device)
            g = self.grid
            if g.curvilinear:
                eng.upload_curvilinear_grid(g.lon, g.lat, g.depth, self._time_s, g.is_spherical(), g.deg2m, g.xdim, g.ydim, g.zdim,
                                            g.get_spatial_hash())  # fmt: skip
            else:
                eng.upload_rectilinear_grid(g.lon, g.lat, g.depth, self._time_s, g.is_spherical(), g.deg2m, g.xdim, g.ydim, g.zdim)
            eng.set_interpolation(INTERP_METHODS[self.vector_interp or ("cgrid_velocity" if g.curvilinear else "linear")], *self.offsets)
            for f in (*(self.vector or ()), *self.fields):
                if f is not None and f._windowed:
                    eng.window_create(f._slot, f.data.dtype, f.data.shape, self.time_window)
                elif f is not None:
                    eng.upload_field(f._slot, f.data)
            self._win[device] = dict(first=0, n=0, resident=set())
            self._engines[device] = eng
        return eng

    def release(self):
        for e in self._engines.values():
            e.close()
        self._engines.clear()


class _ConstantGrid:
    """Grid of the constant fields (reference _core/model.py:292-318): one node, own mesh."""

    def __init__(self, mesh):
        self.mesh = mesh

    def is_spherical(self):
        return self.mesh == "spherical"

    @property
    def deg2m(self):
        return EARTH_RADIUS * np.pi / 180.0 if self.mesh == "spherical" else 1.0


# VectorField.interp_method -> enum pb_interp: XLinear_Velocity, CGrid_Velocity, XFreeslip, XPartialslip
# (reference interpolators/_xinterpolators.py:169-506) and the per-component XNearest (:515-560)
INTERP_METHODS = {"linear": 0, "cgrid_velocity": 1, "freeslip": 2, "partialslip": 3, "nearest": 4}


class FieldSet(_TimeWindow):
    """Velocity fields U, V (, W) laid out (T, Z, Y, X) on one A-grid, plus constant fields.

    Build with :meth:`from_arrays` (NumPy arrays) or ``parcels_b200.adapter.from_parcels`` (a
    FieldSet of the reference package).  Time is float seconds or datetime64/timedelta64.
    """

    def __init__(self, grid: XGrid, U, V, W=None, time=None, interp_method="linear", padding=("low", "low", "high"),
                 time_window=None):  # fmt: skip
        if interp_method not in INTERP_METHODS:
            raise NotImplementedError(f"interp_method {interp_method!r}: this engine has {sorted(INTERP_METHODS)}")
        if grid.curvilinear and interp_method not in ("cgrid_velocity", "linear"):
            raise NotImplementedError("curvilinear grids are supported with CGrid_Velocity and XLinear_Velocity")
        self.interp_method = interp_method
        # time-slab streaming: keep only `time_window` consecutive time levels in HBM (U/V/W may then be any
        # array-like indexable by level: np.memmap, a lazy loader ...); None = every level resident
        self.time_window = None if time_window is None else int(time_window)
        self._win = {}
        # C-grid staggering offsets X, Y, Z: 1 for LOW SGRID padding (reference _xinterpolators.py:99-109)
        self.offsets = tuple(int(p == "low") for p in padding)
        self.grid = grid
        self.fields = {}
        self.constants = {}
        self.context = {}
        self._const_grid = None
        self._extra_grids = []  # _ExtraGrid: scalar fields on grids other than the velocity grid
        self._time_s, self._time_origin = _to_seconds(time)
        for name, arr in (("U", U), ("V", V), ("W", W)):
            if arr is None:
                continue
            if self.time_window is None and not _is_device_array(arr):
                arr = np.asarray(arr)
            if len(arr.shape) != 4:
                raise ValueError(f"{name} must be laid out (T, Z, Y, X); got shape {arr.shape}")
            self.fields[name] = Field(name, arr, grid, self, slot={"U": 0, "V": 1, "W": 2}[name] if self.time_window is None else None,
                                      windowed=self.time_window is not None)  # fmt: skip
        self.U, self.V, self.W = self.fields["U"], self.fields["V"], self.fields.get("W")
        self.UV = VectorField("UV", self.U, self.V)
        self.fields["UV"] = self.UV
        if self.W is not None:
            self.UVW = VectorField("UVW", self.U, self.V, self.W)
            self.fields["UVW"] = self.UVW
        T = self.U.data.shape[0]
        if self._time_s is not None and T != self._time_s.size:
            raise ValueError(f"time axis has {self._time_s.size} levels but U has {T}")
        if self._time_s is None and T != 1:
            raise ValueError("fields with more than one time level need a time axis")
        self._engines: dict[int, Engine] = {}

    @classmethod
    def from_arrays(cls, *, lon, lat, U, V, W=None, depth=None, time=None, mesh="spherical", radius=None,
                    interp_method="linear", padding=("low", "low", "high"), time_window=None, **kw):  # fmt: skip
        return cls(XGrid(lon, lat, depth, mesh=mesh, radius=radius, **kw), U, V, W, time=time, interp_method=interp_method,
                   padding=padding, time_window=time_window)  # fmt: skip

    # -- reference API surface used on this path -----------------------------------------------
    @property
    def time_interval(self):
        """(left, right) in float seconds since the interval start, or None (reference TimeInterval)."""
        if self._time_s is None:
            return None
        return (0.0, float(self._time_s[-1]))

    @property
    def gridset(self):
        return [self.grid] + [x.grid for x in self._extra_grids] + ([self._const_grid] if self._const_grid is not None else [])

    def add_constant_field(self, name, value, mesh="spherical"):
        """reference _core/fieldset.py:175-205."""
        if mesh not in ("flat", "spherical"):
            raise ValueError(f"mesh must be one of ['flat', 'spherical']. Got {mesh!r}.")
        if self._const_grid is None:
            self._const_grid = _ConstantGrid(mesh)
        elif self._const_grid.mesh != mesh:
            raise NotImplementedError("constant fields on two different meshes")
        self.constants[name] = float(np.full((1, 1, 1, 1), value)[0, 0, 0, 0])
        f = Field(name, np.full((1, 1, 1, 1), value), self._const_grid, self, interp_method="constant")
        self.fields[name] = f
        setattr(self, name, f)

    def add_field(self, name, data, interp_method="linear", grid=None, time=None, time_window=None):
        """Scalar field -- in the reference every data variable of the model's dataset is a ``Field`` with its own ``grid`` and
        ``interp_method`` (_core/fieldset.py:89-108, _core/field.py:102-134); here it is added from an array laid out
        (T, Z, Y, X) with T == the time axis, or T == 1 for a field without a time dimension.  ``grid``: an ``XGrid`` other than
        the velocity grid (a second entry of ``fieldset.gridset``; ``time`` = that field's own time axis, default: the
        fieldset's).  Sampled on the device: ``fieldset.<name>[particles]`` / ``.eval(t, z, y, x)``.

        ``time_window=W``: time-slab streaming of this time-varying field -- ``data`` stays the caller's array-like (np.memmap,
        a lazy loader ...) and only ``data[level]`` of the levels entering the window is read.  On the velocity grid W must be
        the FieldSet's ``time_window`` (the field rides on the velocity window); on another grid every windowed field of that
        grid uses one W over the grid's own time axis, slid by the ``eval`` of its fields.  None: the field is uploaded whole."""
        from .engine import Engine

        if interp_method not in Engine.SCALAR_METHODS:
            raise ValueError(f"interp_method must be one of {sorted(Engine.SCALAR_METHODS)}. Got {interp_method!r}")
        if name in self.fields:
            raise ValueError(f"FieldSet already has a Field with name '{name}'")
        if grid is not None and grid is not self.grid:
            return self._add_field_on_grid(name, data, interp_method, grid, time, time_window)
        if self.grid.curvilinear and interp_method not in ("linear", "nearest", "cgrid_tracer"):
            raise NotImplementedError("on curvilinear grids scalar fields are sampled with 'linear' (XLinear), 'cgrid_tracer' (CGrid_Tracer) "
                                      "or 'nearest' (XNearest)")
        if time_window is not None and self.time_window is None:
            raise ValueError(f"{name}: time_window on a FieldSet built without one (FieldSet.from_arrays(..., time_window=W))")
        if time_window is not None and int(time_window) != self.time_window:
            raise ValueError(f"{name}: time_window={time_window}, but a field on the velocity grid streams through the "
                             f"FieldSet's window of {self.time_window} levels")  # fmt: skip
        data = _field_data(name, data, time_window)
        nt = 1 if self._time_s is None else self._time_s.size
        if data.shape[0] not in (1, nt) or tuple(data.shape[1:]) != tuple(self.U.data.shape[1:]):
            raise ValueError(f"{name} has shape {data.shape}; expected ({nt} or 1, {', '.join(map(str, self.U.data.shape[1:]))})")
        slot = 3 + sum(1 for f in self.fields.values() if isinstance(f, Field) and f._host is None and f._slot is not None and f._slot >= 3)
        f = Field(name, data, self.grid, self, interp_method=interp_method, slot=slot, windowed=time_window is not None)
        self.fields[name] = f
        setattr(self, name, f)
        if f._windowed:
            self._window_add_field(slot, data)
        else:
            for eng in self._engines.values():
                eng.upload_field(slot, data)
        return f

    def _add_field_on_grid(self, name, data, interp_method, grid, time, time_window):
        if not isinstance(grid, XGrid):
            raise TypeError(f"grid must be an XGrid, got {type(grid).__name__}")
        if grid.curvilinear and interp_method not in ("linear", "nearest", "cgrid_tracer"):
            raise NotImplementedError("on curvilinear grids scalar fields are sampled with 'linear', 'cgrid_tracer' or 'nearest'")
        data = _field_data(name, data, time_window)
        time_s = self._time_s if time is None else _to_seconds(time)[0]
        nt = 1 if time_s is None else time_s.size
        nz = 1 if grid.depth is None else len(grid.depth)
        ny, nx = (grid.lon.shape if grid.curvilinear else (len(grid.lat), len(grid.lon)))
        if data.shape[0] not in (1, nt) or data.shape[1] not in (1, nz) or data.shape[2:] != (ny, nx):
            raise ValueError(f"{name} has shape {data.shape}; expected ({nt} or 1, {nz} or 1, {ny}, {nx}) on its grid")
        host = next((x for x in self._extra_grids if x.grid is grid), None)
        if host is None:
            host = _ExtraGrid(grid, time_s)
            self._extra_grids.append(host)
        elif (host._time_s is None) != (time_s is None) or (time_s is not None and not np.array_equal(host._time_s, time_s)):
            raise NotImplementedError("fields on one grid share one time axis")
        if len(host.fields) >= 13:
            raise NotImplementedError("at most 13 scalar fields per grid")
        if time_window is not None:
            host.use_window(name, time_window)
        f = Field(name, data, grid, self, interp_method=interp_method, slot=3 + len(host.fields), host=host,
                  windowed=time_window is not None)  # fmt: skip
        host.fields.append(f)
        self.fields[name] = f
        setattr(self, name, f)
        if f._windowed:
            host._window_add_field(f._slot, data)
        else:
            for eng in host._engines.values():
                eng.upload_field(f._slot, data)
        return f

    def add_vector_field(self, name, U, V, W=None, *, grid, interp_method="linear", padding=("low", "low", "high"), time=None,
                         time_window=None):  # fmt: skip
        """A further VectorField on ANOTHER XGrid of the FieldSet (reference: any ``VectorField(name, U, V[, W])`` of the fieldset,
        e.g. a wind field on the atmospheric model's grid, _core/field.py:205-248), for sampling in user kernels --
        ``fieldset.<name>[particles]`` / ``.eval(t, z, y, x)`` -> (u, v[, w]) in the units ``fieldset.UV`` gives (degrees per second on
        a spherical mesh).  The advection kernels keep using ``fieldset.UV`` / ``UVW`` on the velocity grid.
        ``time_window=W``: the components stream through the grid's window of W levels, as in :meth:`add_field`."""
        if not isinstance(grid, XGrid) or grid is self.grid:
            raise ValueError("add_vector_field needs an XGrid other than the velocity grid (fieldset.UV is the vector field of that one)")
        if name in self.fields:
            raise ValueError(f"FieldSet already has a Field with name '{name}'")
        if interp_method not in INTERP_METHODS or (grid.curvilinear and interp_method not in ("cgrid_velocity", "linear")):
            raise NotImplementedError(f"interp_method {interp_method!r} on this grid")
        time_s = self._time_s if time is None else _to_seconds(time)[0]
        host = next((x for x in self._extra_grids if x.grid is grid), None)
        if host is None:
            host = _ExtraGrid(grid, time_s)
            self._extra_grids.append(host)
        elif host.vector is not None:
            raise NotImplementedError("one vector field per grid")
        elif host._engines:
            raise NotImplementedError("add the vector field of a grid before its fields are first sampled")
        if time_window is not None:
            host.use_window(name, time_window)
        comps = []
        for cname, arr in (("U", U), ("V", V), ("W", W)):
            if arr is None:
                comps.append(None)
                continue
            if time_window is not None:
                _field_data(f"{name}.{cname}", arr, time_window)
            else:
                arr = np.ascontiguousarray(arr)
                if arr.ndim != 4 or arr.dtype not in (np.float32, np.float64):
                    raise ValueError(f"{name}.{cname} must be a float32 / float64 array laid out (T, Z, Y, X)")
            comps.append(Field(f"{name}_{cname}", arr, grid, self, interp_method="linear", slot=len(comps), host=host,
                               windowed=time_window is not None))  # fmt: skip
        host.vector, host.vector_interp = tuple(comps), interp_method
        host.offsets = tuple(int(p == "low") for p in padding)
        vf = VectorField(name, comps[0], comps[1], comps[2], host=host)
        self.fields[name] = vf
        setattr(self, name, vf)
        return vf

    def add_context(self, name, value):
        """reference _core/fieldset.py:207-222; the value is then also an attribute (``fieldset.<name>``, :101-108)."""
        if not isinstance(name, str) or not name.isidentifier():
            raise ValueError(f"Expected a string that is a valid Python variable name, got {name!r}")
        if name in self.context:
            raise ValueError(f"FieldSet already has a context with name '{name}'")
        self.context[name] = value

    def __getattr__(self, name):
        """Context variables as attributes, as user kernels read them (``fieldset.dres``; reference _core/fieldset.py:101-108)."""
        ctx = self.__dict__.get("context")
        if ctx is not None and name in ctx:
            return ctx[name]
        raise AttributeError(f"FieldSet has no attribute '{name}'")

    # -- engine management: fields are uploaded once and stay resident in HBM --------------------
    def engine(self, device: int = 0) -> Engine:
        eng = self._engines.get(device)
        if eng is None:
            eng = Engine(device)
            g = self.grid
            if g.curvilinear:
                eng.upload_curvilinear_grid(g.lon, g.lat, g.depth, self._time_s, g.is_spherical(), g.deg2m, g.xdim, g.ydim,
                                            g.zdim, g.get_spatial_hash())  # fmt: skip
            else:
                eng.upload_rectilinear_grid(g.lon, g.lat, g.depth, self._time_s, g.is_spherical(), g.deg2m, g.xdim, g.ydim, g.zdim)
            eng.set_interpolation(INTERP_METHODS[self.interp_method], *self.offsets)
            for slot, name in enumerate(("U", "V", "W")):
                if name in self.fields:
                    d = self.fields[name].data
                    if _is_device_array(d):
                        # already in HBM (e.g. a torch CUDA tensor): attached without a copy, kept alive by the engine
                        cai = d.__cuda_array_interface__
                        if cai.get("strides") is not None or cai["typestr"] not in ("<f4", "<f8"):
                            raise ValueError(f"device field {name} must be C-contiguous float32/float64 (T, Z, Y, X)")
                        eng.attach_field_device(slot, int(cai["data"][0]), cai["typestr"] == "<f8", tuple(cai["shape"]), keepalive=d)
                    elif self.time_window is None:
                        eng.upload_field(slot, d)
                    else:
                        eng.window_create(slot, d.dtype, d.shape, self.time_window)
            for f in self.fields.values():
                if isinstance(f, Field) and f._host is None and f._slot is not None and f._slot >= 3:
                    if f._windowed:
                        eng.window_create(f._slot, f.data.dtype, f.data.shape, self.time_window)
                    else:
                        eng.upload_field(f._slot, f.data)
            self._win[device] = dict(first=0, n=0, resident=set())
            self._engines[device] = eng
        return eng

    # -- time-slab streaming (_TimeWindow): U, V, W and the scalar fields added with time_window ------------------------------
    def _windowed_fields(self):
        uvw = [(slot, self.fields[name].data) for slot, name in enumerate(("U", "V", "W")) if name in self.fields]
        return uvw + [(f._slot, f.data) for f in self.fields.values() if isinstance(f, Field) and f._host is None and f._slot is not None
                      and f._slot >= 3 and f._windowed]  # fmt: skip

    def release(self):
        for e in self._engines.values():
            e.close()
        self._engines.clear()
        for x in self._extra_grids:
            x.release()
