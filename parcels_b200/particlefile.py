"""Trajectory output: ``ParticleFile`` with the reference's constructor / ``write`` / ``close`` API
(``_core/particlefile.py:54-190``), Parquet through pyarrow exactly as the reference writes it.

What differs is where the row selection happens.  While a ``ParticleSet`` is resident in HBM (between the
output intervals of one ``execute`` call), ``write`` asks the device for the rows the reference's
``_to_write_particles`` rule (``:198-221``) selects and copies back ONLY those rows of the written columns
(``pb_output_select`` / ``pb_output_gather``); the Parquet encoding stays on the host, unchanged.
"""

from __future__ import annotations

import datetime
from pathlib import Path

import numpy as np

__all__ = ["ParticleFile", "read_particlefile", "to_write_particles"]


def to_write_particles(particle_data, t):
    """Host form of the selection rule (reference ``_to_write_particles``, _core/particlefile.py:198-221):
    rows with finite ``t`` and ``t - |dt/2| <= particles.t <= t + |dt/2|`` (or ``dt`` NaN and equal times)."""
    pt, pdt = particle_data["t"], particle_data["dt"]
    fin = np.isfinite(pt)
    with np.errstate(invalid="ignore"):
        near = (t - np.abs(pdt / 2) <= pt) & (t + np.abs(pdt / 2) >= pt)
        exact = np.isnan(pdt) & (t == pt)
    return np.where((near | exact) & fin & np.isfinite(particle_data["particle_id"]))[0]


def _cf_time_attrs(origin):
    """Units of the ``t`` column (reference _core/utils/time.py:88-120): seconds since the interval's left edge."""
    if not isinstance(origin, np.datetime64):  # float / timedelta64 time axes: plain seconds
        return {"units": "seconds"}
    ts = np.datetime64(origin, "us").astype(datetime.datetime)
    return {"units": f"seconds since {ts.strftime('%Y-%m-%d %H:%M:%S')}", "calendar": "gregorian"}


class ParticleFile:
    def __init__(self, path, outputdt, compression="zstd", mode=None):
        if not isinstance(outputdt, (np.timedelta64, datetime.timedelta, float)):
            raise ValueError(f"Expected outputdt to be a np.timedelta64, datetime.timedelta or float (in seconds), got {type(outputdt)}")
        self._compression = compression
        if isinstance(outputdt, datetime.timedelta):
            outputdt = outputdt.total_seconds()
        elif isinstance(outputdt, np.timedelta64):
            outputdt = float(outputdt / np.timedelta64(1, "s"))
        path = Path(path)
        if path.suffix != ".parquet":
            raise ValueError(f"ParticleFile data is stored in Parquet files - file extension must be '.parquet'. Got {path.suffix=!r}.")
        if outputdt <= 0:
            raise ValueError(f"outputdt must be positive/non-zero. Got {outputdt=!r}")
        if mode not in {None, "w"}:
            raise ValueError(f"Invalid mode value {mode!r}. Expected one of None or 'w'.")
        if path.exists():
            if mode is None:
                raise ValueError(f"Path '{path}' already exists. Use mode='w' or use a new path.")
            path.unlink()
        if not path.parent.exists():
            raise ValueError(f"Folder location for '{path} does not exist. Create the folder location first.")
        self._outputdt = outputdt
        self._path = path
        self._writer = None
        self.metadata = {}
        self.rows_written = 0
        self.device_writes = 0  # writes whose rows were selected and compacted on the GPU

    outputdt = property(lambda self: self._outputdt)
    path = property(lambda self: self._path)

    def set_metadata(self, parcels_grid_mesh):
        from . import __version__

        self.metadata.update({"feature_type": "trajectory", "Conventions": "CF-1.6/CF-1.7",
                              "ncei_template_version": "NCEI_NetCDF_Trajectory_Template_v2.0",
                              "parcels_version": f"parcels_b200 {__version__}", "parcels_grid_mesh": repr(parcels_grid_mesh)})  # fmt: skip

    def _schema(self, pclass, fieldset):
        import pyarrow as pa

        fields = []
        for v in pclass.written_variables():
            attrs = dict(v.attrs)
            if v.name == "t" and fieldset.time_interval is not None:
                attrs.update(_cf_time_attrs(fieldset._time_origin))
            fields.append(pa.field(v.name, pa.from_numpy_dtype(v.dtype), metadata={str(k): str(a) for k, a in attrs.items()}))
        return pa.schema(fields, metadata={str(k): str(a) for k, a in self.metadata.items()})

    def write(self, pset, t, fieldset=None, indices=None):
        """Write the rows of ``pset`` that are due at time ``t`` (seconds, or a time object of the fieldset)."""
        import pyarrow as pa
        import pyarrow.parquet as pq

        fieldset = fieldset if fieldset is not None else pset.fieldset
        pclass = pset._pclass
        if self._writer is None:
            # Same schema, values and compression as the reference's writer (:155-160).  Dictionary encoding is kept
            # for `t` only (few distinct values per write): attempting it on the float position columns and the
            # ids is what dominates pyarrow's encode time and never pays off there.
            self._writer = pq.ParquetWriter(self.path, self._schema(pclass, fieldset), compression=self._compression,
                                            use_dictionary=["t"])
        if isinstance(t, np.datetime64):
            t = float((t - fieldset._time_origin) / np.timedelta64(1, "s"))
        elif isinstance(t, np.timedelta64):
            t = float(t / np.timedelta64(1, "s"))
        names = [v.name for v in pclass.written_variables()]
        cols, on_device = pset._output_columns(float(t), names, indices)
        self.device_writes += int(on_device)
        self.rows_written += len(cols[names[0]]) if names else 0
        self._writer.write_table(pa.table({n: pa.array(cols[n]) for n in names}, schema=self._writer.schema))

    def close(self):
        if self._writer is not None:
            self._writer.close()
            self._writer = None

    def __enter__(self):
        return self

    def __exit__(self, *args):
        self.close()


def read_particlefile(path):
    """The written table as a dict of NumPy columns (the reference returns a pandas DataFrame, :224-262)."""
    import pyarrow.parquet as pq

    tab = pq.read_table(path)
    return {n: tab.column(n).to_numpy() for n in tab.column_names}
