"""Host-side mirror of the reference's sequential-filter orbit determination surface for the batched GPU path
(SURVEY.md §8 (f)-2, BASELINE configs[4]).  Reference paths are relative to /root/reference/nyx-core/src:

* ``GroundStation``            od/ground_station/{mod.rs:47-75, builtin.rs:25-117, trk_device.rs:35-253}
* ``MeasurementType``          od/msr/types.rs:31-45
* ``TrackingDataArc``          od/msr/trackingdata (epochs + tracker + data per type), reduced to arrays
* ``ProcessNoise3D``           od/snc.rs:38-56, 118-134, 288-311
* ``SigmaRejection``           od/process/rejectcrit.rs:35-46
* ``KfEstimate``               od/estimate/kfestimate.rs (nominal state, covariance, state deviation)
* ``SpacecraftUncertainty``    od/estimate/sc_uncertainty.rs:36-138
* ``KalmanODProcess``          od/process/{initializers.rs:60-113, mod.rs:128-497}; `predict_until` / `predict_for` mod.rs:440-496;
                               `SpacecraftKalmanOD` = MsrSize 2,
                               `SpacecraftKalmanScalarOD` = MsrSize 1 (od/mod.rs:77-91)
* ``InterlinkTxSpacecraft``    od/interlink/{trk_device.rs:37-260, sensitivity.rs:50-172}: spacecraft-to-spacecraft range and Doppler
                               through ``nyxb_od_interlink_batch``
* ``BatchLeastSquares``        od/blse/mod.rs:30-541 (``BLSSolver``, ``BLSSolution``; `estimate` / `evaluate` through
                               ``nyxb_od_bls_batch`` / ``nyxb_od_bls_evaluate_batch``, n problems in one launch)

Nothing here runs the filter: ``KalmanODProcess.process_arcs`` packs the ensemble into the SoA arrays of
``nyxb_od_ekf_batch`` (include/nyxb.h) — ONE kernel launch runs every filter from the first to the last measurement
(propagation with the STM, time updates, measurement updates, state replacement) on the device.  There is no CPU
fallback.  The measurement *simulator* (`simulate_tracking`, stands in for od/simulator/arc.rs) is host-side data
generation for tests and the benchmark, not part of the filter path.
"""
from __future__ import annotations

import enum
import math
from dataclasses import dataclass, field, replace
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import abi
from .cosmic import Orbit, Spacecraft, duration_to_seconds
from .dynamics import _rotation_c
from .frames import IAU_EARTH_FRAME, NS_PER_S, Almanac, Frame


class MeasurementType(enum.IntEnum):
    Range = abi.MSR_RANGE
    Doppler = abi.MSR_DOPPLER
    Azimuth = abi.MSR_AZIMUTH      # degrees, ground stations (GroundStation.with_msr_type)
    Elevation = abi.MSR_ELEVATION
    X = abi.MSR_X          # position fixes (PositionDevice), km in the integration frame
    Y = abi.MSR_Y
    Z = abi.MSR_Z


_POSITION_TYPES = (MeasurementType.X, MeasurementType.Y, MeasurementType.Z)
# the observation slots of an arc for ground stations that measure angles (nyxb_od_aer_batch): slot = type
AER_TYPES = (MeasurementType.Range, MeasurementType.Doppler, MeasurementType.Azimuth, MeasurementType.Elevation)
_ANGLE_TYPES = (MeasurementType.Azimuth, MeasurementType.Elevation)


class KalmanVariant(enum.IntEnum):
    ReferenceUpdate = abi.KF_REFERENCE_UPDATE      # EKF
    DeviationTracking = abi.KF_DEVIATION_TRACKING  # CKF


class LocalFrame(enum.IntEnum):
    Inertial = 0
    RIC = 1
    VNC = 2


class ODError(RuntimeError):
    pass


@dataclass(frozen=True)
class StochasticNoise:
    """`StochasticNoise` reduced to what the filter reads: the white-noise sigma (covariance = sigma^2,
    noise/white.rs) and the constant part of the bias (trk_device.rs:238-253)."""

    sigma: float
    bias_constant: float = 0.0

    def covariance(self, _epoch_ns: int = 0) -> float:
        return self.sigma ** 2

    @classmethod
    def default_range_km(cls) -> "StochasticNoise":
        return cls(2e-3)     # noise/mod.rs: 2 m

    @classmethod
    def default_doppler_km_s(cls) -> "StochasticNoise":
        return cls(3e-6)     # noise/mod.rs: 3 mm/s


@dataclass
class GroundStation:
    name: str
    latitude_deg: float
    longitude_deg: float
    height_km: float
    frame: Frame = IAU_EARTH_FRAME
    elevation_mask_deg: float = 0.0
    measurement_types: Sequence[MeasurementType] = (MeasurementType.Range, MeasurementType.Doppler)
    stochastic_noises: Dict[MeasurementType, StochasticNoise] = field(default_factory=lambda: {
        MeasurementType.Range: StochasticNoise.default_range_km(), MeasurementType.Doppler: StochasticNoise.default_doppler_km_s()})
    integration_time: Optional[int] = None
    light_time_correction: bool = False

    # builtin.rs:25-117
    @classmethod
    def dss65_madrid(cls, elevation_mask_deg, range_noise_km: StochasticNoise, doppler_noise_km_s: StochasticNoise):
        return cls("Madrid", 40.427_222, 4.250_556, 0.834_939, IAU_EARTH_FRAME, elevation_mask_deg,
                   stochastic_noises={MeasurementType.Range: range_noise_km, MeasurementType.Doppler: doppler_noise_km_s})

    @classmethod
    def dss34_canberra(cls, elevation_mask_deg, range_noise_km: StochasticNoise, doppler_noise_km_s: StochasticNoise):
        return cls("Canberra", -35.398_333, 148.981_944, 0.691_750, IAU_EARTH_FRAME, elevation_mask_deg,
                   stochastic_noises={MeasurementType.Range: range_noise_km, MeasurementType.Doppler: doppler_noise_km_s})

    @classmethod
    def dss13_goldstone(cls, elevation_mask_deg, range_noise_km: StochasticNoise, doppler_noise_km_s: StochasticNoise):
        return cls("Goldstone", 35.247_164, 243.205, 1.071_149_04, IAU_EARTH_FRAME, elevation_mask_deg,
                   stochastic_noises={MeasurementType.Range: range_noise_km, MeasurementType.Doppler: doppler_noise_km_s})

    def with_msr_type(self, msr_type: MeasurementType, noise: StochasticNoise) -> "GroundStation":
        """`GroundStation::with_msr_type` (ground_station/mod.rs:137-150): sets the type's noise and appends the type to the list
        unless it is there already."""
        msr_type = MeasurementType(msr_type)
        self.stochastic_noises = {**self.stochastic_noises, msr_type: noise}
        if msr_type not in self.measurement_types:
            self.measurement_types = [*self.measurement_types, msr_type]
        return self

    @property
    def has_angles(self) -> bool:
        return any(t in _ANGLE_TYPES for t in self.measurement_types)

    def north_east_fixed(self):
        """Unit geodetic north and east in the body-fixed frame (the S and E axes of the SEZ frame, Vallado's RAZEL)."""
        lat, lon = math.radians(self.latitude_deg), math.radians(self.longitude_deg)
        north = np.array([-math.sin(lat) * math.cos(lon), -math.sin(lat) * math.sin(lon), math.cos(lat)])
        east = np.array([-math.sin(lon), math.cos(lon), 0.0])
        return north, east

    def body_fixed(self):
        """Geodetic (lat, long, height) -> body-fixed Cartesian position and local zenith on the frame's ellipsoid
        (anise `Orbit::try_latlongalt`; sphere when the frame has no polar radius)."""
        a = self.frame.mean_equatorial_radius_km()
        b = self.frame.polar_radius_km if self.frame.polar_radius_km is not None else a
        e2 = 1.0 - (b * b) / (a * a)
        lat, lon = math.radians(self.latitude_deg), math.radians(self.longitude_deg)
        sl, cl = math.sin(lat), math.cos(lat)
        nu = a / math.sqrt(1.0 - e2 * sl * sl)
        pos = np.array([(nu + self.height_km) * cl * math.cos(lon), (nu + self.height_km) * cl * math.sin(lon),
                        (nu * (1.0 - e2) + self.height_km) * sl])
        up = np.array([cl * math.cos(lon), cl * math.sin(lon), sl])
        return pos, up

    def to_c(self, integration_frame: Frame, almanac: Optional[Almanac]) -> abi.GroundStationC:
        if self.integration_time is not None or self.light_time_correction:
            raise ODError("only instantaneous measurements without light-time correction are supported on the GPU path")
        types = list(self.measurement_types)
        if not 1 <= len(types) <= 2 or len(set(types)) != len(types):
            raise ODError("a ground station carries one or two of {Range, Doppler}")
        return self._fill_c(abi.GroundStationC(), types, integration_frame, almanac)

    def to_aer_c(self, integration_frame: Frame, almanac: Optional[Almanac]) -> abi.AerStationC:
        """The station for nyxb_od_aer_batch: one to four distinct types of Range, Doppler, Azimuth and Elevation."""
        if self.integration_time is not None or self.light_time_correction:
            raise ODError("only instantaneous measurements without light-time correction are supported on the GPU path")
        types = list(self.measurement_types)
        if not 1 <= len(types) <= 4 or len(set(types)) != len(types) or any(t not in AER_TYPES for t in types):
            raise ODError("a ground station carries one to four distinct types of {Range, Doppler, Azimuth, Elevation}")
        g = self._fill_c(abi.AerStationC(), types, integration_frame, almanac)
        north, east = self.north_east_fixed()
        for i in range(3):
            g.north_fixed[i] = north[i]
            g.east_fixed[i] = east[i]
        return g

    def _fill_c(self, g, types, integration_frame: Frame, almanac: Optional[Almanac]):
        pos, up = self.body_fixed()
        for i in range(3):
            g.pos_fixed_km[i] = pos[i]
            g.up_fixed[i] = up[i]
        g.elevation_mask_deg = self.elevation_mask_deg
        g.rot = _rotation_c(self.frame.rotation)
        if self.frame.ephemeris_id == integration_frame.ephemeris_id:
            g.body = abi.NYXB_CENTRAL_BODY
            g.body_radius_km = -1.0   # same body: the elevation mask is the only visibility test (trk_device.rs:162-166)
        else:
            if almanac is None:
                raise ODError("an almanac with the station's body is needed when it does not sit on the integration centre")
            g.body = almanac.body_index(self.frame.ephemeris_id)
            g.body_radius_km = integration_frame.mean_equatorial_radius_km()
        g.n_types = len(types)
        for i, t in enumerate(types):
            if t not in self.stochastic_noises:
                raise ODError(f"NoiseNotConfigured: {t.name}")
            g.types[i] = int(t)
            g.noise_var[i] = self.stochastic_noises[t].covariance()
            g.bias[i] = self.stochastic_noises[t].bias_constant
        return g


@dataclass
class PositionDevice:
    """`PositionDevice` (od/position/mod.rs): GNSS-style position fixes, X, Y and Z of the spacecraft in the integration frame of the
    estimate.  `with_noise(type, noise)` adds the type to the device's list (in call order) with its noise, as the reference builds it.
    The filter measures the component at the type's LIST position and differentiates the type's own component (see
    nyxb_position_device in include/nyxb.h); a bias cancels in the computed observation."""

    name: str
    measurement_types: List[MeasurementType] = field(default_factory=list)
    stochastic_noises: Dict[MeasurementType, StochasticNoise] = field(default_factory=dict)

    def with_noise(self, msr_type: MeasurementType, noise: StochasticNoise) -> "PositionDevice":
        msr_type = MeasurementType(msr_type)
        self.stochastic_noises[msr_type] = noise
        if msr_type not in self.measurement_types:
            self.measurement_types.append(msr_type)
        return self

    def to_c(self) -> abi.PositionDeviceC:
        types = list(self.measurement_types)
        if not 1 <= len(types) <= 3 or len(set(types)) != len(types) or any(t not in _POSITION_TYPES for t in types):
            raise ODError("a position device carries one to three distinct types of {X, Y, Z}")
        d = abi.PositionDeviceC()
        d.n_types = len(types)
        for i, t in enumerate(types):
            d.types[i] = int(t)
            d.noise_var[i] = self.stochastic_noises[t].covariance()
            d.bias[i] = self.stochastic_noises[t].bias_constant
        return d


@dataclass
class InterlinkTxSpacecraft:
    """`InterlinkTxSpacecraft` (od/interlink/trk_device.rs:37-260): a transmitter spacecraft known by its recorded trajectory `traj`,
    measuring the range and Doppler of the filtered spacecraft (the receiver).  The filter runs through nyxb_od_interlink_batch, with
    the reference's as-coded quirks (include/nyxb.h, nyxb_interlink_tx): the computed Doppler ignores the transmitter's velocity, the
    sensitivity rows use the observed range and Doppler, and an epoch outside `traj` ends the filter.  Only instantaneous measurements
    without aberration correction, with `traj` in the integration frame of the estimates."""

    traj: "Traj"
    measurement_types: Sequence[MeasurementType]
    stochastic_noises: Dict[MeasurementType, StochasticNoise]
    integration_time: Optional[int] = None
    ab_corr: Optional[object] = None

    def name(self) -> str:
        """trk_device.rs:93-95: the trajectory's name, or "unnamed"."""
        return self.traj.name if self.traj.name is not None else "unnamed"

    def to_c(self, tx: int, integration_frame: Frame) -> abi.InterlinkTxC:
        """The device for nyxb_od_interlink_batch, its transmitter in column `tx` of the recordings."""
        if self.integration_time is not None:
            raise ODError("interlink: integrated (two-way) measurements are not supported on the GPU path")
        if self.ab_corr is not None:
            raise ODError("interlink: aberration correction is not supported on the GPU path (ab_corr must be None)")
        fr = self.traj.template.orbit.frame
        if fr.ephemeris_id != integration_frame.ephemeris_id or fr.rotation != integration_frame.rotation:
            raise ODError(f"interlink: the transmitter's trajectory is in {fr.name}, the estimates in {integration_frame.name}")
        if len(self.traj) == 0:
            raise ODError("interlink: the transmitter's trajectory is empty")
        types = [MeasurementType(t) for t in self.measurement_types]
        if not 1 <= len(types) <= 2 or len(set(types)) != len(types) or any(t not in (MeasurementType.Range, MeasurementType.Doppler)
                                                                               for t in types):
            raise ODError("an interlink carries one or two of {Range, Doppler}")
        d = abi.InterlinkTxC()
        d.tx = int(tx)
        d.n_types = len(types)
        for i, t in enumerate(types):
            if t not in self.stochastic_noises:
                raise ODError(f"NoiseNotConfigured: {t.name}")
            d.types[i] = int(t)
            d.noise_var[i] = self.stochastic_noises[t].covariance()
            d.bias[i] = self.stochastic_noises[t].bias_constant
        try:
            d.body_radius_km = integration_frame.mean_equatorial_radius_km()
        except ValueError as e:
            raise ODError(f"interlink: the line-of-sight test needs the radius of the integration frame's body ({e})") from None
        return d


def interlink_sink(trajs: Sequence["Traj"]):
    """The transmitter recordings of nyxb_od_interlink_batch: (TrajSink, n_tx, arrays kept alive), column j = trajs[j], ascending."""
    n_tx = len(trajs)
    cap = max((len(t) for t in trajs), default=0)
    epoch = np.zeros((cap, n_tx), dtype=np.int64)
    state = np.zeros((6, cap, n_tx))
    count = np.zeros(n_tx, dtype=np.int64)
    for j, t in enumerate(trajs):
        k = len(t)
        epoch[:k, j] = t.epochs_ns
        state[:, :k, j] = np.asarray(t.states, dtype=np.float64)[:, :6].T
        count[j] = k
    sink = abi.TrajSink(cap, epoch.ctypes.data, state.ctypes.data, count.ctypes.data)
    return sink, n_tx, (epoch, state, count)


@dataclass
class TrackingDataArc:
    """One tracking schedule (epochs + tracker names) with `n` observation sets: obs[k][type][i], NaN = type not in
    the measurement's data (both NaN: measurement k absent from arc i).  `types` names the observation slots: (Range, Doppler),
    (X, Y, Z) for position fixes, whose obs is [m][3][n] (all three NaN: absent), or AER_TYPES (Range, Doppler, Azimuth, Elevation)
    for ground stations with angles, whose obs is [m][4][n]."""

    epoch_ns: np.ndarray            # [m] int64 ascending
    tracker: List[str]              # [m]
    obs: np.ndarray                 # [m][len(types)][n] float64
    types: Sequence[MeasurementType] = (MeasurementType.Range, MeasurementType.Doppler)

    @property
    def is_position(self) -> bool:
        return tuple(self.types) == _POSITION_TYPES

    @property
    def is_aer(self) -> bool:
        return tuple(self.types) == AER_TYPES

    def __post_init__(self):
        self.epoch_ns = np.ascontiguousarray(self.epoch_ns, dtype=np.int64)
        self.obs = np.ascontiguousarray(self.obs, dtype=np.float64)
        self.types = tuple(MeasurementType(t) for t in self.types)
        m = self.epoch_ns.shape[0]
        if self.obs.ndim == 2:
            self.obs = np.ascontiguousarray(self.obs[:, :, None])
        if self.types not in ((MeasurementType.Range, MeasurementType.Doppler), _POSITION_TYPES, AER_TYPES):
            raise ODError("types must be (Range, Doppler), (X, Y, Z) or (Range, Doppler, Azimuth, Elevation)")
        if self.is_aer:
            if len(self.tracker) != m or self.obs.shape[0] != m or self.obs.shape[1] != 4:
                raise ODError("expected epoch_ns[m], tracker[m], obs[m][4][n]")
        elif self.is_position:
            if len(self.tracker) != m or self.obs.shape[0] != m or self.obs.shape[1] != 3:
                raise ODError("expected epoch_ns[m], tracker[m], obs[m][3][n]")
        elif len(self.tracker) != m or self.obs.shape[0] != m or self.obs.shape[1] != 2:
            raise ODError("expected epoch_ns[m], tracker[m], obs[m][2][n]")
        if m and np.any(np.diff(self.epoch_ns) < 0):
            raise ODError("measurement epochs must be ascending")

    def __len__(self):
        return self.epoch_ns.shape[0]

    @property
    def n(self) -> int:
        return self.obs.shape[2]

    # ---- parquet I/O in the reference's layout (od/msr/trackingdata/io_parquet.rs:43-354): one arc per file
    _COLUMNS = ("Range (km)", "Doppler (km/s)")   # MeasurementType::to_field names (od/msr/types.rs)
    _POS_COLUMNS = ("X (km)", "Y (km)", "Z (km)")
    _AER_COLUMNS = ("Range (km)", "Doppler (km/s)", "Azimuth (deg)", "Elevation (deg)")

    def to_parquet(self, path, index: int = 0, metadata: Optional[dict] = None):
        """`TrackingDataArc::to_parquet` for the observation set `index`: "Epoch (UTC)", "Tracking device" and one nullable
        Float64 column per measurement type present; measurements absent from this arc are not written."""
        import pyarrow as pa
        import pyarrow.parquet as pq

        from .cosmic import epochs_to_utc_iso

        o = self.obs[:, :, index]
        present = ~np.isnan(o).all(axis=1)
        if not present.any():
            raise ODError("EmptyDataset: tracking data arc to parquet")
        cols = [pa.array(epochs_to_utc_iso(self.epoch_ns[present]), type=pa.string()),
                pa.array([t for t, p in zip(self.tracker, present) if p], type=pa.string())]
        fields = [pa.field("Epoch (UTC)", pa.string(), nullable=False), pa.field("Tracking device", pa.string(), nullable=False)]
        for c, name in enumerate(self._POS_COLUMNS if self.is_position else self._AER_COLUMNS if self.is_aer else self._COLUMNS):
            v = o[present, c]
            if np.isnan(v).all():
                continue   # unique_types(): a type no measurement carries has no column
            cols.append(pa.array(v, type=pa.float64(), mask=np.isnan(v)))
            fields.append(pa.field(name, pa.float64(), nullable=True, metadata={"unit": name[name.index("(") + 1:-1]}))
        meta = {"Purpose": "Tracking Arc Data"}
        meta.update(metadata or {})
        pq.write_table(pa.Table.from_arrays(cols, schema=pa.schema(fields, metadata=meta)), str(path))
        return path

    @classmethod
    def from_parquet(cls, path, types=None) -> "TrackingDataArc":
        """`TrackingDataArc::from_parquet` (io_parquet.rs:43-213): needs "Epoch (UTC)", "Tracking device" and at least one of
        the measurement columns this path knows: range / Doppler, or X / Y / Z (an arc of types (X, Y, Z)), not both kinds; rows are
        sorted by epoch.  `types=AER_TYPES` reads range, Doppler, "Azimuth (deg)" and "Elevation (deg)" into an arc of those four
        types instead."""
        import pyarrow.parquet as pq

        tab = pq.read_table(str(path))
        names = set(tab.column_names)
        for need in ("Epoch (UTC)", "Tracking device"):
            if need not in names:
                raise ODError(f"MissingData: {need}")
        if types is not None:
            if tuple(MeasurementType(t) for t in types) != AER_TYPES:
                raise ODError("from_parquet reads types=None or types=AER_TYPES")
            if names & set(cls._POS_COLUMNS):
                raise ODError("X / Y / Z columns in an arc of ground-station types")
            if not names & set(cls._AER_COLUMNS):
                raise ODError("MissingData: `Range (km)`, `Doppler (km/s)`, `Azimuth (deg)` or `Elevation (deg)`")
            return cls._read_columns(tab, names, cls._AER_COLUMNS, AER_TYPES)
        ground, pos = bool(names & set(cls._COLUMNS)), bool(names & set(cls._POS_COLUMNS))
        if ground and pos:
            raise ODError("range / Doppler and X / Y / Z columns in one arc: one tracker kind per arc")
        if not ground and not pos:
            raise ODError("MissingData: `Range (km)`, `Doppler (km/s)` or `X (km)`, `Y (km)`, `Z (km)`")
        types = _POSITION_TYPES if pos else (MeasurementType.Range, MeasurementType.Doppler)
        return cls._read_columns(tab, names, cls._POS_COLUMNS if pos else cls._COLUMNS, types)

    @classmethod
    def _read_columns(cls, tab, names, columns, types) -> "TrackingDataArc":
        from .cosmic import utc_iso_to_epochs

        ep = utc_iso_to_epochs(tab["Epoch (UTC)"].to_pylist())
        obs = np.full((len(ep), len(columns)), np.nan)
        for c, name in enumerate(columns):
            if name in names:
                obs[:, c] = [np.nan if v is None else v for v in tab[name].to_pylist()]
        order = np.argsort(ep, kind="stable")
        trk = tab["Tracking device"].to_pylist()
        return cls(ep[order], [trk[i] for i in order], obs[order][:, :, None], types)

    def filter_by_offset(self, start_ns: Optional[int] = None, end_ns: Optional[int] = None) -> "TrackingDataArc":
        """`TrackingDataArc::filter_by_offset` (od/msr/trackingdata/mod.rs:394-410) as coded: the measurements in
        [first + start, first + end), first being the first epoch of the schedule.  Whatever the bound kind, the end is exclusive, and
        an open end stands for the last epoch, so that the last measurement is dropped; an open start keeps from the first."""
        if len(self) == 0:
            return self
        first, last = int(self.epoch_ns[0]), int(self.epoch_ns[-1])
        lo = first if start_ns is None else first + int(start_ns)
        hi = last if end_ns is None else first + int(end_ns)
        keep = (self.epoch_ns >= lo) & (self.epoch_ns < hi)
        return TrackingDataArc(self.epoch_ns[keep], [t for t, k in zip(self.tracker, keep) if k], self.obs[keep], self.types)

    @classmethod
    def stack(cls, arcs: Sequence["TrackingDataArc"]) -> "TrackingDataArc":
        """n single-observation-set arcs -> one arc with n observation sets over the union of their schedules (what
        `process_arcs` takes); a (epoch, tracker) pair missing from an arc is NaN there."""
        keys = sorted({(int(e), t) for a in arcs for e, t in zip(a.epoch_ns, a.tracker)})
        pos = {k: i for i, k in enumerate(keys)}
        n = sum(a.n for a in arcs)
        types = arcs[0].types if arcs else (MeasurementType.Range, MeasurementType.Doppler)
        if any(a.types != types for a in arcs):
            raise ODError("arcs of different measurement types")
        obs = np.full((len(keys), len(types), n), np.nan)
        col = 0
        for a in arcs:
            rows = [pos[(int(e), t)] for e, t in zip(a.epoch_ns, a.tracker)]
            obs[rows, :, col:col + a.n] = a.obs
            col += a.n
        return cls(np.array([k[0] for k in keys], dtype=np.int64), [k[1] for k in keys], obs, types)


@dataclass(frozen=True)
class SigmaRejection:
    num_sigmas: float = 3.0


@dataclass
class ProcessNoise3D:
    diag: np.ndarray
    disable_time: int
    local_frame: Optional[LocalFrame] = None

    def __post_init__(self):
        # the SNC packing (config_c) knows RIC and inertial only; it would treat any other frame as inertial
        if self.local_frame is not None and self.local_frame not in (LocalFrame.Inertial, LocalFrame.RIC):
            raise ODError(f"process noise in the {LocalFrame(self.local_frame).name} frame is not supported (RIC or inertial)")

    @classmethod
    def from_diagonal(cls, values, disable_time: int, local_frame: Optional[LocalFrame] = None):
        v = np.asarray(values, dtype=np.float64)
        assert v.shape == (3,), "Not enough values for the size of the SNC matrix"
        return cls(v, int(disable_time), local_frame)

    @classmethod
    def from_velocity_km_s(cls, velocity_noise, noise_duration: int, disable_time: int, local_frame: Optional[LocalFrame] = None):
        """snc.rs:288-311: diag = velocity noise / noise duration (seconds)."""
        return cls(np.asarray(velocity_noise, dtype=np.float64) / duration_to_seconds(noise_duration), int(disable_time), local_frame)


def dcm_ric_to_inertial(orbit: Orbit) -> np.ndarray:
    """Columns R, I, C (anise `Orbit::dcm_to_inertial(LocalFrame::RIC)`): R = r/|r|, C = h/|h|, I = C x R."""
    r, v = orbit.radius_km, orbit.velocity_km_s
    rh = r / np.linalg.norm(r)
    h = np.cross(r, v)
    ch = h / np.linalg.norm(h)
    ih = np.cross(ch, rh)
    return np.column_stack([rh, ih, ch])


def dcm_vnc_to_inertial(orbit: Orbit) -> np.ndarray:
    """Columns V, N, C (anise `Orbit::dcm_to_inertial(LocalFrame::VNC)`): V = v/|v|, N = h/|h|, C = V x N; the convention of the
    targeter's correction frame (nyx_b200/csrc/nyxb_target.h)."""
    r, v = orbit.radius_km, orbit.velocity_km_s
    vh = v / np.linalg.norm(v)
    h = np.cross(r, v)
    nh = h / np.linalg.norm(h)
    return np.column_stack([vh, nh, np.cross(vh, nh)])


@dataclass
class KfEstimate:
    nominal_state: Spacecraft
    covar: np.ndarray                       # [9][9]
    state_deviation: np.ndarray = field(default_factory=lambda: np.zeros(9))

    @classmethod
    def from_covar(cls, nominal_state: Spacecraft, covar) -> "KfEstimate":
        return cls(nominal_state, np.array(covar, dtype=np.float64).reshape(9, 9))

    @classmethod
    def from_diag(cls, nominal_state: Spacecraft, diag) -> "KfEstimate":
        return cls(nominal_state, np.diag(np.asarray(diag, dtype=np.float64)))

    def state(self) -> Spacecraft:
        """nominal + deviation (`Spacecraft + OVector<9>`, cosmic/spacecraft.rs:713-728: Cr clamped to [0, 2])."""
        v = self.nominal_state.to_vector() + self.state_deviation
        v[6] = min(max(v[6], 0.0), 2.0)
        return self.nominal_state.with_vector(self.nominal_state.epoch(), v)

    def to_random_variable(self):
        """`KfEstimate::to_random_variable` (od/estimate/kfestimate.rs:157-160): the multivariate normal of this estimate, centred on
        the nominal state shifted by the state deviation (what a Monte Carlo of the estimate draws from)."""
        from .monte_carlo import MvnSpacecraft

        return MvnSpacecraft.from_spacecraft_cov(self.nominal_state, self.covar, mean=self.state_deviation)


@dataclass
class SpacecraftUncertainty:
    """sc_uncertainty.rs:36-138 (defaults included).  As coded the covariance is rotated as D^T C D with D = the
    local->inertial state DCM (RIC or VNC); the rotation-rate block of the local state DCM is taken as zero here (anise's
    `rot_mat_dt` is not in the tree)."""

    nominal: Spacecraft
    frame: Optional[LocalFrame] = None
    x_km: float = 0.5
    y_km: float = 0.5
    z_km: float = 0.5
    vx_km_s: float = 50e-5
    vy_km_s: float = 50e-5
    vz_km_s: float = 50e-5
    coeff_reflectivity: float = 0.0
    coeff_drag: float = 0.0
    mass_kg: float = 0.0

    def to_estimate(self) -> KfEstimate:
        vals = [self.x_km, self.y_km, self.z_km, self.vx_km_s, self.vy_km_s, self.vz_km_s, self.coeff_reflectivity,
                self.coeff_drag, self.mass_kg]
        if any(v < 0.0 for v in vals):
            raise ODError("uncertainties must be positive")
        if self.frame == LocalFrame.RIC:
            d3 = dcm_ric_to_inertial(self.nominal.orbit)
        elif self.frame == LocalFrame.VNC:
            d3 = dcm_vnc_to_inertial(self.nominal.orbit)
        else:
            d3 = np.eye(3)
        d6 = np.zeros((6, 6))
        d6[:3, :3] = d3
        d6[3:, 3:] = d3
        cov = np.zeros((9, 9))
        cov[:6, :6] = d6.T @ np.diag(np.square(vals[:6])) @ d6
        for i in range(6, 9):
            cov[i, i] = vals[i] ** 2
        return KfEstimate.from_covar(self.nominal, cov)


_STATE_ITEMS = ("X", "Y", "Z", "Vx", "Vy", "Vz", "Cr", "Cd", "Mass")
_STATE_UNITS = ("km", "km", "km", "km/s", "km/s", "km/s", "unitless", "unitless", "kg")


def _state_columns(cols, schema, est, tmpl: Spacecraft, fields=None):
    """The state-parameter columns of the OD exports (export.rs:159-171, 385-395): est [9][k] estimated states; a parameter the
    state cannot give is left out."""
    import pyarrow as pa

    from .param import EXPORT_PARAMS, StateError, evaluate

    frame = tmpl.orbit.frame
    for f in (EXPORT_PARAMS if fields is None else fields):
        try:
            vals = evaluate(f, est[:6], frame.mu_km3_s2(), tmpl, cr=est[6], cd=est[7], prop_mass_kg=est[8])
        except StateError:
            continue
        cols.append(pa.array(vals, type=pa.float64()))
        schema.append(pa.field(str(f), pa.float64(), nullable=False, metadata={"unit": f.unit, "Frame": frame.name}))


def _sigma_columns(cols, schema, diag, frame_name: str):
    """"Sigma <item> (<frame>) (<unit>)" from the covariance diagonal, diag [k][n_items] (export.rs:235-243, 428-435)."""
    import pyarrow as pa

    sig = np.sqrt(np.maximum(diag, 0.0))
    for q in range(diag.shape[1]):
        cols.append(pa.array(sig[:, q], type=pa.float64()))
        schema.append(pa.field(f"Sigma {_STATE_ITEMS[q]} ({frame_name}) ({_STATE_UNITS[q]})", pa.float64(), nullable=False))


def _cov_units():
    """Units of the upper-triangle covariance entries, row by row, as export.rs:186-215 assigns them."""
    units = []
    for i in range(9):
        for j in range(i, 9):
            if i < 3:
                u = "km^2" if j < 3 else ("km^2/s" if j < 6 else ("km*kg" if j == 8 else "km"))
            elif i < 6:
                u = "km^2/s^2" if j < 6 else ("km/s*kg" if j == 8 else "km/s")
            elif i == 8 or j == 8:
                u = "kg^2"
            else:
                u = "unitless"
            units.append(u)
    return units


def _estimate_columns(epochs, est, cov, tmpl: Spacecraft, fields=None):
    """The per-estimate columns the OD exports share (export.rs:159-246, 385-446): "Epoch (UTC)", the state parameters of
    estimate.state() est [9][k], the 45 "Covariance <a>*<b> (<frame>) (<unit>)" entries of cov [k][9][9], "Sigma <item> (<frame>)
    (<unit>)" and "Sigma <item> (RIC) (<unit>)".  The RIC sigmas follow the as-coded product D C D^T with D = the RIC->inertial state
    DCM of estimate.state(), its rate block taken as zero (as SpacecraftUncertainty)."""
    import pyarrow as pa

    from .cosmic import epochs_to_utc_iso

    k = est.shape[1]
    frame = tmpl.orbit.frame
    cols = [pa.array(epochs_to_utc_iso(np.asarray(epochs, dtype=np.int64)), type=pa.string())]
    schema = [pa.field("Epoch (UTC)", pa.string(), nullable=False)]
    _state_columns(cols, schema, est, tmpl, fields)
    units = _cov_units()
    q = 0
    for a in range(9):
        for b in range(a, 9):
            cols.append(pa.array(cov[:, a, b], type=pa.float64()))
            schema.append(pa.field(f"Covariance {_STATE_ITEMS[a]}*{_STATE_ITEMS[b]} ({frame.name}) ({units[q]})", pa.float64(),
                                   nullable=False))
            q += 1
    _sigma_columns(cols, schema, np.diagonal(cov, axis1=1, axis2=2), frame.name)
    ric = np.empty((k, 6))
    for j in range(k):
        d3 = dcm_ric_to_inertial(Orbit(*[float(v) for v in est[:6, j]], 0, frame))
        d6 = np.zeros((6, 6))
        d6[:3, :3] = d3
        d6[3:, 3:] = d3
        ric[j] = np.diag(d6 @ cov[j, :6, :6] @ d6.T)
    _sigma_columns(cols, schema, ric, "RIC")
    return cols, schema


@dataclass
class ODSolution:
    """Results of n filters: final estimates and the per-measurement residual records (od/process/solution)."""

    final_state_soa: np.ndarray      # [9][n]
    final_epoch_ns: np.ndarray       # [n]
    covar: np.ndarray                # [n][9][9]
    state_deviation: np.ndarray      # [9][n]
    resid_ratio: np.ndarray          # [m][2][n]
    prefit: np.ndarray               # [m][2][n]
    postfit: np.ndarray              # [m][2][n]
    msr_flags: np.ndarray            # [m][n]
    est_state: Optional[np.ndarray]  # [m][9][n]
    est_covar_diag: Optional[np.ndarray]
    details: np.ndarray
    status: np.ndarray
    templates: Sequence[Spacecraft] = ()
    arc: Optional["TrackingDataArc"] = None
    devices: Optional[Dict[str, GroundStation]] = None
    # every estimate (ODSolution.estimates) when run with an estimates capacity K: epoch / tag [K][n], nominal / deviation [K][9][n],
    # covar / stm [K][81][n] ((r, c) at [k][c*9 + r][i]), count [n] (see nyxb_od_records in include/nyxb.h)
    records: Optional[dict] = None
    process: Optional["KalmanODProcess"] = None
    initial_estimates: Optional[Sequence[KfEstimate]] = None
    # set on the solution smooth() returns: state / deviation / fs_ratio [K][9][n], covar [K][81][n], postfit [K][2][n] by estimate
    # position, status [n], and the filter's own postfit [m][2][n]
    smoother: Optional[dict] = None

    def accepted(self) -> np.ndarray:
        return ((self.msr_flags & abi.MSRF_PROCESSED) != 0) & ((self.msr_flags & abi.MSRF_REJECTED) == 0)

    def rejected(self) -> np.ndarray:
        return (self.msr_flags & abi.MSRF_REJECTED) != 0

    def final_estimate(self, i: int) -> KfEstimate:
        sc = self.templates[i].with_vector(int(self.final_epoch_ns[i]), self.final_state_soa[:, i])
        return KfEstimate(sc, self.covar[i].copy(), self.state_deviation[:, i].copy())

    def _to_parquet_estimates(self, path, index, fields, metadata):
        import pyarrow as pa
        import pyarrow.parquet as pq

        L = self.n_estimates(index)
        if L == 0:
            raise ODError("EmptyDataset: no estimate recorded")
        tmpl = self.templates[index]
        ests = [self.estimate(k, index) for k in range(L)]
        est = np.stack([e.state().to_vector() for e in ests], axis=1)          # [9][L]
        cov = np.stack([e.covar for e in ests])                                # [L][9][9]
        cols, schema = _estimate_columns(self.records["epoch"][:L, index], est, cov, tmpl, fields)
        res = self.residuals(index)
        M = self.process.msr_size if self.process is not None else 2
        rec = self.records
        tracker = [None] * L
        types = [None] * L
        for p in range(L):
            src = p + 1 if (self.smoother is not None and p < L - 1) else p
            if res[p] is None:
                continue
            mk, w, _, _ = self._tag_fields(int(rec["tag"][src, index]))
            key = self.arc.tracker[mk] if self.arc is not None else None
            tracker[p] = self._tracker_name(key) if key is not None else None
            dev = (self.devices or {}).get(key)
            tl = list(dev.measurement_types) if dev is not None else [MeasurementType.Range, MeasurementType.Doppler]
            types[p] = [int(t) for t in tl[w * M:(w + 1) * M]]
        for label, j in (("Prefit residual", 0), ("Postfit residual", 1)):
            for mt, un in self._residual_types():
                v = np.full(L, np.nan)
                for p in range(L):
                    if res[p] is not None and int(mt) in types[p]:
                        v[p] = res[p][j][types[p].index(int(mt))]
                cols.append(pa.array(v, type=pa.float64(), mask=np.isnan(v)))
                schema.append(pa.field(f"{label}: {mt.name} ({un})", pa.float64(), nullable=True))
        ratio = np.array([r[2] if r is not None else np.nan for r in res])
        cols.append(pa.array(ratio, type=pa.float64(), mask=np.isnan(ratio)))
        schema.append(pa.field("Residual ratio", pa.float64(), nullable=True))
        cols.append(pa.array([r[3] if r is not None else None for r in res], type=pa.bool_()))
        schema.append(pa.field("Residual Rejected", pa.bool_(), nullable=True))
        cols.append(pa.array(tracker, type=pa.string()))
        schema.append(pa.field("Tracker", pa.string(), nullable=True))
        for it in _STATE_ITEMS:                          # the gains are not kept (None on a smoother run, as the reference)
            for j in range(M):
                cols.append(pa.nulls(L, type=pa.float64()))
                schema.append(pa.field(f"Gain {it}*[{j}]", pa.float64(), nullable=True))
        units = _cov_units()
        fs = self.filter_smoother_ratios(index)
        for a in range(9):                               # as coded: the first nine covariance units (export.rs:333-343)
            v = fs[:, a] if fs is not None else np.full(L, np.nan)
            mask = np.arange(L) == L - 1 if fs is not None else np.ones(L, dtype=bool)   # a NaN ratio itself is Some(NaN)
            cols.append(pa.array(v, type=pa.float64(), mask=mask))
            schema.append(pa.field(f"Filter-smoother ratio {_STATE_ITEMS[a]} ({units[a]})", pa.float64(), nullable=True))
        meta = {"Purpose": "Orbit determination results"}
        meta.update(metadata or {})
        pq.write_table(pa.Table.from_arrays(cols, schema=pa.schema(schema, metadata=meta)), str(path))
        return path

    # ---- estimates, smoothing and statistics (od/process/solution/{mod,smooth,stats}.rs)
    def _is_position(self) -> bool:
        return self.arc is not None and self.arc.is_position

    def _is_aer(self) -> bool:
        return self.arc is not None and self.arc.is_aer

    def _tag_fields(self, tag):
        """(measurement, window, rejected, msr_size) of a record tag, in the layout of the run's tracker kind (NYXB_OD_TAG, or
        NYXB_OD_POS_TAG for position fixes and stations with angles)."""
        return abi.od_pos_tag_fields(tag) if self._is_position() or self._is_aer() else abi.od_tag_fields(tag)

    def _ratio_slot(self, w: int, M: int) -> int:
        """The slot of window w's residual ratio: w for stations with angles, else w at msr_size 1 and 0 otherwise."""
        return w if (M == 1 or self._is_aer()) else 0

    def _residual_types(self):
        """(type, unit) of the residual columns: Range / Doppler (and Azimuth / Elevation for stations with angles), or X / Y / Z for
        position fixes."""
        if self._is_position():
            return [(t, "km") for t in _POSITION_TYPES]
        rd = [(MeasurementType.Range, "km"), (MeasurementType.Doppler, "km/s")]
        return rd + [(MeasurementType.Azimuth, "deg"), (MeasurementType.Elevation, "deg")] if self._is_aer() else rd

    def _tracker_name(self, key: str) -> str:
        """The "Tracker" of a residual: the device's name, which for an interlink is its trajectory's name (export.rs)."""
        dev = (self.devices or {}).get(key)
        return dev.name() if isinstance(dev, InterlinkTxSpacecraft) else key

    def _need_records(self):
        if self.records is None:
            raise ODError("no estimate records: run process_arcs(.., estimates_capacity=K)")
        return self.records

    def n_estimates(self, i: int) -> int:
        """Number of stored estimates of filter i (the reference's `estimates.len()` when nothing was truncated)."""
        rec = self._need_records()
        return int(min(rec["count"][i], rec["epoch"].shape[0]))

    def is_smoother_run(self) -> bool:
        return self.smoother is not None

    def error(self, i: int) -> Optional[str]:
        """None, or why filter i (or its smoothing) failed."""
        st = int(self.smoother["status"][i]) if self.smoother is not None else int(self.status[i])
        if st == 0:
            return None
        names = {abi.ERR_TOO_FEW_MEASUREMENTS: "TooFewMeasurements: fewer than two estimates",
                 abi.ERR_SINGULAR_STM: "SingularStateTransitionMatrix", abi.ERR_RECORDS_TRUNCATED: "estimate records truncated",
                 abi.ERR_EPHEMERIS: "epoch outside ephemeris coverage",
                 abi.ERR_TX_NO_DATA: "ODTrajError: the interlink transmitter's trajectory does not cover the epoch",
                 abi.ERR_NO_RANGE: "MeasurementSimError: Range measurement data is missing"}
        return names.get(st, f"status {st}")

    def estimate(self, k: int, i: int) -> KfEstimate:
        """Estimate k of filter i (smoothed on a smoother run): nominal state, covariance and state deviation."""
        rec = self._need_records()
        if not 0 <= k < self.n_estimates(i):
            raise IndexError(k)
        src = self.smoother if self.smoother is not None else rec
        sc = self.templates[i].with_vector(int(rec["epoch"][k, i]), rec["nominal"][k, :, i])
        return KfEstimate(sc, src["covar"][k, :, i].reshape(9, 9).T.copy(), src["deviation"][k, :, i].copy())

    def filter_smoother_ratios(self, i: int) -> Optional[np.ndarray]:
        """[k][9] filter-smoother ratios of filter i on a smoother run (the last row, None in the reference, is NaN)."""
        if self.smoother is None:
            return None
        return self.smoother["fs_ratio"][: self.n_estimates(i), :, i].copy()

    def residuals(self, i: int) -> List[Optional[tuple]]:
        """`self.residuals` of filter i, one entry per estimate: None for a time update (and, smoothed, a successor without residual
        or an invisible smoothed state), else (prefit[M], postfit[M], ratio, rejected).  On a smoother run position k holds the
        residual of estimate k+1 with its postfit recomputed at estimate k, and the last position the filter's own (as coded)."""
        rec = self._need_records()
        M = self.process.msr_size if self.process is not None else 2
        L = self.n_estimates(i)
        filt_post = self.smoother["filter_postfit"] if self.smoother is not None else self.postfit
        out = []
        for p in range(L):
            src = p + 1 if (self.smoother is not None and p < L - 1) else p
            tag = int(rec["tag"][src, i])
            if tag < 0:
                out.append(None)
                continue
            mk, w, rej, _ = self._tag_fields(tag)
            slots = [w * M + q for q in range(M)]
            if src != p:
                post = self.smoother["postfit"][p, slots, i]
                if np.isnan(post).all():
                    out.append(None)
                    continue
            else:
                post = filt_post[mk, slots, i]
            out.append((self.prefit[mk, slots, i].copy(), np.array(post), float(self.resid_ratio[mk, self._ratio_slot(w, M), i]), bool(rej)))
        return out

    def _rms(self, i, f):
        res = self.residuals(i)
        if not res:
            return float("nan")
        return float(np.sqrt(sum(f(r) for r in res if r is not None) / len(res)))

    def rms_prefit_residuals(self, i: int = 0) -> float:
        """stats.rs:148-155: the denominator counts every estimate (time updates too)."""
        return self._rms(i, lambda r: float(r[0] @ r[0]))

    def rms_postfit_residuals(self, i: int = 0) -> float:
        """stats.rs:157-164 (a sigma-rejected filter residual has a NaN postfit, as in the reference)."""
        return self._rms(i, lambda r: float(r[1] @ r[1]))

    def rms_residual_ratios(self, i: int = 0) -> float:
        """stats.rs:166-173."""
        return self._rms(i, lambda r: r[2] ** 2)

    def smooth(self) -> "ODSolution":
        """`ODSolution::smooth` (od/process/solution/smooth.rs:104-249) of all n filters in ONE launch; returns a new solution (the
        reference consumes `self`) whose estimates are the smoothed ones, with filter-smoother ratios, the smoothed postfit residuals
        (`residuals(i)`; in the per-measurement `postfit` array, measurement of estimate p >= 1 gets the value of position p - 1, the
        first estimate's measurement NaN), prefit and ratios kept, no gains.  Needs complete records: when a filter produced more
        estimates than the capacity, the filters are run once more with a capacity of max(count) first.  Per-filter failures (filter
        status, fewer than two estimates, singular STM) are in `error(i)`; they never abort the batch."""
        rec = self._need_records()
        if self.process is None or self.arc is None:
            raise ODError("smooth() needs the solution of KalmanODProcess.process_arcs")
        if self.smoother is not None:
            raise ODError("already smoothed")
        cap = rec["epoch"].shape[0]
        if int(rec["count"].max(initial=0)) > cap:
            again = self.process.process_arcs(self.initial_estimates, self.arc, record_estimates=self.est_state is not None,
                                              estimates_capacity=int(rec["count"].max()))
            return again.smooth()
        odp = self.process
        frame = self.templates[0].orbit.frame
        eng = odp.prop.engine(frame, odp.almanac)
        pos = odp.is_position
        if pos:
            names, dev_c = odp.position_devices_c()
            tracker = np.array([names.index(t) if t in names else -1 for t in self.arc.tracker], dtype=np.int32)
            sm = eng.od_position_smooth_batch(odp.config_c(), len(names), dev_c, tracker, self.arc.obs, rec, self.status)
        elif odp.is_interlink:
            names, dev_c, sink = odp.interlink_c(frame)
            tracker = np.array([names.index(t) if t in names else -1 for t in self.arc.tracker], dtype=np.int32)
            sm = eng.od_interlink_smooth_batch(odp.config_c(), len(names), dev_c, sink, tracker, self.arc.obs, rec, self.status)
        elif self.arc.is_aer:
            names, st_c = odp.aer_stations_c(frame)
            tracker = np.array([names.index(t) if t in names else -1 for t in self.arc.tracker], dtype=np.int32)
            sm = eng.od_aer_smooth_batch(odp.config_c(), len(names), st_c, tracker, self.arc.obs, rec, self.status)
        else:
            names, st_c = odp.stations_c(frame)
            tracker = np.array([names.index(t) if t in names else -1 for t in self.arc.tracker], dtype=np.int32)
            sm = eng.od_smooth_batch(odp.config_c(), len(names), st_c, tracker, self.arc.obs, rec, self.status)
        sm["filter_postfit"] = self.postfit
        post = np.full(self.postfit.shape, np.nan)
        M = odp.msr_size
        for i in range(len(self.status)):
            if sm["status"][i] != 0:
                continue
            for p in range(self.n_estimates(i) - 1):
                tag = int(rec["tag"][p + 1, i])
                if tag >= 0:
                    mk, w, _, _ = self._tag_fields(tag)
                    post[mk, w * M:(w + 1) * M, i] = sm["postfit"][p, w * M:(w + 1) * M, i]
        return replace(self, postfit=post, smoother=sm)

    def to_parquet(self, path, index: int = 0, fields=None, metadata: Optional[dict] = None):
        """`ODSolution::to_parquet` (od/process/solution/export.rs:60-688) for filter `index`.

        With estimate records (`process_arcs(.., estimates_capacity=K)`), one row per estimate as export.rs writes it: "Epoch (UTC)",
        the state parameters of estimate.state(), the 45 covariance entries, the sigmas in the state frame and in RIC (the column code
        of PredictionSolution.to_parquet), prefit / postfit residuals per measurement type, "Residual ratio", "Residual Rejected",
        "Tracker" (null for an estimate without residual), the gains (null: not kept) and the filter-smoother ratios (set on a
        smoother run, null otherwise and on the last estimate).  A smoother run exports the smoothed estimates with their
        (off-by-one, as coded) residuals.

        Without records, one row per processed measurement epoch from the per-measurement outputs: "Epoch (UTC)", the state
        parameters of the estimate, "Sigma <item> (<frame>) (<unit>)" from the covariance diagonal, the residuals, ratio, rejection and
        tracker; that needs `process_arcs(.., record_estimates=True)` and carries no off-diagonal covariance terms."""
        import pyarrow as pa
        import pyarrow.parquet as pq

        from .cosmic import epochs_to_utc_iso

        if self.records is not None:
            return self._to_parquet_estimates(path, index, fields, metadata)

        if self.est_state is None or self.est_covar_diag is None or self.arc is None:
            raise ODError("no per-measurement estimates recorded: run process_arcs(.., record_estimates=True)")
        rows = np.nonzero((self.msr_flags[:, index] & abi.MSRF_PROCESSED) != 0)[0]
        if len(rows) == 0:
            raise ODError("EmptyDataset: no measurement was processed")
        tmpl = self.templates[index]
        frame = tmpl.orbit.frame
        est = self.est_state[rows, :, index].T          # [9][k]
        cols = [pa.array(epochs_to_utc_iso(self.arc.epoch_ns[rows]), type=pa.string())]
        schema = [pa.field("Epoch (UTC)", pa.string(), nullable=False)]
        _state_columns(cols, schema, est, tmpl, fields)
        _sigma_columns(cols, schema, self.est_covar_diag[rows, :, index], frame.name)
        # residual slots follow the order of the tracker's measurement types (include/nyxb.h: nyxb_od_outputs)
        ns = self.prefit.shape[1]
        slot_type = np.full((len(rows), ns), -1)
        for a, r in enumerate(rows):
            dev = (self.devices or {}).get(self.arc.tracker[r])
            types = list(dev.measurement_types) if dev is not None else [MeasurementType.Range, MeasurementType.Doppler]
            slot_type[a, :len(types)] = [int(t) for t in types]
        for label, arr in (("Prefit residual", self.prefit), ("Postfit residual", self.postfit)):
            for mt, un in self._residual_types():
                v = np.full(len(rows), np.nan)
                for q in range(ns):
                    hit = slot_type[:, q] == int(mt)
                    v[hit] = arr[rows[hit], q, index]
                cols.append(pa.array(v, type=pa.float64(), mask=np.isnan(v)))
                schema.append(pa.field(f"{label}: {mt.name} ({un})", pa.float64(), nullable=True))
        ratio = self.resid_ratio[rows, 0, index]
        for q in range(1, ns):
            ratio = np.where(np.isnan(ratio), self.resid_ratio[rows, q, index], ratio)
        cols.append(pa.array(ratio, type=pa.float64(), mask=np.isnan(ratio)))
        schema.append(pa.field("Residual ratio", pa.float64(), nullable=True))
        cols.append(pa.array((self.msr_flags[rows, index] & abi.MSRF_REJECTED) != 0, type=pa.bool_()))
        schema.append(pa.field("Residual Rejected", pa.bool_(), nullable=True))
        cols.append(pa.array([self._tracker_name(self.arc.tracker[r]) for r in rows], type=pa.string()))
        schema.append(pa.field("Tracker", pa.string(), nullable=True))
        meta = {"Purpose": "Orbit determination results"}
        meta.update(metadata or {})
        pq.write_table(pa.Table.from_arrays(cols, schema=pa.schema(schema, metadata=meta)), str(path))
        return path


@dataclass
class PredictionSolution:
    """Results of n covariance predictions (`KalmanODProcess::predict_until`, od/process/mod.rs:440-486): the final estimates and
    the records of the time updates.  Record k of run i sits at epoch0_ns[i] + k * max_step_ns; record 0 is the initial estimate.
    rec_count[i] records were produced; the first min(rec_count[i], capacity) are stored."""

    final_state_soa: np.ndarray          # [9][n] nominal state
    final_epoch_ns: np.ndarray           # [n]
    covar: np.ndarray                    # [n][9][9]
    state_deviation: np.ndarray          # [9][n]
    details: np.ndarray
    status: np.ndarray
    rec_count: np.ndarray                # [n]
    rec_state: Optional[np.ndarray]      # [K][9][n] estimate.state() (nominal + deviation)
    rec_covar: Optional[np.ndarray]      # [K][81][n], (r, c) at [k][c*9 + r][i]
    epoch0_ns: np.ndarray                # [n]
    max_step_ns: int
    templates: Sequence[Spacecraft] = ()

    @property
    def capacity(self) -> int:
        for a in (self.rec_state, self.rec_covar):
            if a is not None:
                return a.shape[0]
        return 0

    def stored(self, i: int) -> int:
        return int(min(self.rec_count[i], self.capacity))

    def record_epochs(self, i: int) -> np.ndarray:
        """Epochs of the stored records of run i."""
        return self.epoch0_ns[i] + np.arange(self.stored(i), dtype=np.int64) * self.max_step_ns

    def record_covar(self, k: int, i: int) -> np.ndarray:
        return self.rec_covar[k, :, i].reshape(9, 9).T.copy()

    def final_estimate(self, i: int) -> KfEstimate:
        sc = self.templates[i].with_vector(int(self.final_epoch_ns[i]), self.final_state_soa[:, i])
        return KfEstimate(sc, self.covar[i].copy(), self.state_deviation[:, i].copy())

    def to_parquet(self, path, index: int = 0, fields=None, metadata: Optional[dict] = None, msr_size: int = 2):
        """`ODSolution::to_parquet` (od/process/solution/export.rs:60-470) of the solution `predict_until` returns, which has no
        measurement types, for run `index`: "Epoch (UTC)", the state parameters of estimate.state() (default
        `Spacecraft::export_params`), the 45 "Covariance <a>*<b> (<frame>) (<unit>)" entries, "Sigma <item> (<frame>) (<unit>)",
        "Sigma <item> (RIC) (<unit>)", then the residual, gain and filter-smoother columns, all null.  The RIC sigmas follow the
        as-coded product D C D^T with D = the RIC->inertial state DCM of estimate.state() (export.rs:430-446), its rate block taken
        as zero (as SpacecraftUncertainty).  The per-element sigma columns of orbital-element parameters are not written."""
        import pyarrow as pa
        import pyarrow.parquet as pq

        if self.rec_state is None or self.rec_covar is None:
            raise ODError("records of both states and covariances are needed: predict with a record capacity")
        k = self.stored(index)
        if k == 0:
            raise ODError("TooFewMeasurements: need 1 estimate to export")
        tmpl = self.templates[index]
        est = self.rec_state[:k, :, index].T                                   # [9][k]
        cov = self.rec_covar[:k, :, index].reshape(k, 9, 9).transpose(0, 2, 1)   # [k][r][c]
        cols, schema = _estimate_columns(self.record_epochs(index), est, cov, tmpl, fields)
        units = _cov_units()

        def nulls(name, typ):
            cols.append(pa.nulls(k, type=typ))
            schema.append(pa.field(name, typ, nullable=True))

        for j in range(msr_size):
            nulls(f"Whitened residual #{j}", pa.float64())
        nulls("Residual ratio", pa.float64())
        nulls("Residual Rejected", pa.bool_())
        nulls("Tracker", pa.string())
        for it in _STATE_ITEMS:                          # no measurement types: len 0 != MsrSize::DIM (export.rs:302-331)
            for j in range(msr_size):
                nulls(f"Gain {it}*[{j}]", pa.float64())
        for a in range(9):                               # as coded: the first nine covariance units (export.rs:333-343)
            nulls(f"Filter-smoother ratio {_STATE_ITEMS[a]} ({units[a]})", pa.float64())
        meta = {"Purpose": "Orbit determination results"}
        meta.update(metadata or {})
        pq.write_table(pa.Table.from_arrays(cols, schema=pa.schema(schema, metadata=meta)), str(path))
        return path


class KalmanODProcess:
    """`KalmanODProcess<SpacecraftDynamics, MsrSize, 3, GroundStation>` (od/process/mod.rs) on the batched GPU path."""

    def __init__(self, prop, kf_variant: KalmanVariant, sigma_reject: Optional[SigmaRejection], devices: Dict[str, GroundStation],
                 almanac: Optional[Almanac], msr_size: int = 2):
        self.prop = prop
        self.kf_variant = kf_variant
        self.sigma_reject = sigma_reject
        self.devices = dict(devices)
        self.almanac = almanac
        self.process_noise: List[ProcessNoise3D] = []
        self.max_step = 60 * NS_PER_S            # initializers.rs:71
        self.epoch_precision = 1_000             # 1 microsecond, initializers.rs:72
        self.msr_size = int(msr_size)

    new = classmethod(lambda cls, *a, **k: cls(*a, **k))

    def with_process_noise(self, snc: ProcessNoise3D) -> "KalmanODProcess":
        self.process_noise = [snc]
        return self

    # ---- packing
    def config_c(self) -> abi.OdConfigC:
        if len(self.process_noise) > 1:
            raise ODError("one process-noise model is supported on the GPU path")
        if self.max_step <= 0:
            raise ODError(f"StepSize: {self.max_step}")
        c = abi.OdConfigC()
        c.variant = int(self.kf_variant)
        c.msr_size = self.msr_size
        c.reject_num_sigmas = self.sigma_reject.num_sigmas if self.sigma_reject is not None else -1.0
        c.max_step_ns = int(self.max_step)
        c.epoch_precision_ns = int(self.epoch_precision)
        if self.process_noise:
            snc = self.process_noise[0]
            c.snc_enabled = 1
            c.snc_frame = 1 if snc.local_frame == LocalFrame.RIC else 0
            for i in range(3):
                c.snc_diag[i] = float(snc.diag[i])
            c.snc_disable_time_ns = int(snc.disable_time)
        return c

    def _kinds(self):
        kinds = {type(d) for d in self.devices.values()}
        if len(kinds) > 1:
            raise ODError("mixed tracker kinds: all devices must be GroundStations, all PositionDevices or all InterlinkTxSpacecraft")
        return kinds

    @property
    def is_position(self) -> bool:
        """True for a filter over PositionDevices; the reference's `Trk` is one type, so the kinds are never mixed."""
        return self._kinds() == {PositionDevice}

    @property
    def is_interlink(self) -> bool:
        """True for a filter over InterlinkTxSpacecraft (never mixed with another kind)."""
        return self._kinds() == {InterlinkTxSpacecraft}

    def interlink_c(self, frame: Frame):
        """(names, devices, recordings) for nyxb_od_interlink_batch: one recording column per distinct trajectory."""
        names = list(self.devices)
        trajs: List = []
        arr = (abi.InterlinkTxC * max(len(names), 1))()
        for i, nme in enumerate(names):
            t = self.devices[nme].traj
            col = next((j for j, u in enumerate(trajs) if u is t), None)
            if col is None:
                col = len(trajs)
                trajs.append(t)
            arr[i] = self.devices[nme].to_c(col, frame)
        return names, arr, interlink_sink(trajs)

    def position_devices_c(self):
        names = list(self.devices)
        arr = (abi.PositionDeviceC * max(len(names), 1))()
        for i, nme in enumerate(names):
            arr[i] = self.devices[nme].to_c()
        return names, arr

    def stations_c(self, frame: Frame):
        names = list(self.devices)
        arr = (abi.GroundStationC * max(len(names), 1))()
        for i, nme in enumerate(names):
            arr[i] = self.devices[nme].to_c(frame, self.almanac)
        return names, arr

    def aer_stations_c(self, frame: Frame):
        names = list(self.devices)
        arr = (abi.AerStationC * max(len(names), 1))()
        for i, nme in enumerate(names):
            arr[i] = self.devices[nme].to_aer_c(frame, self.almanac)
        return names, arr

    def process_arcs(self, initial_estimates: Sequence[KfEstimate], arc: TrackingDataArc, record_estimates: bool = False,
                     estimates_capacity: Optional[int] = None) -> ODSolution:
        """n independent `process_arc(initial_estimate_i, arc_i)` runs (od/process/mod.rs:128-497) in one launch.  With
        `estimates_capacity` K, the first K entries of each filter's ODSolution.estimates are recorded (1 456 bytes each), which
        `ODSolution.smooth()`, `residuals`, the RMS statistics and the per-estimate parquet export need; the filter's results do not
        change.  Ground stations run through nyxb_od_aer_batch exactly when the arc's types are AER_TYPES (range, Doppler, azimuth,
        elevation); stations that measure angles need such an arc.  InterlinkTxSpacecraft devices run through
        nyxb_od_interlink_batch over a (Range, Doppler) arc."""
        n = len(initial_estimates)
        if arc.n != n:
            raise ODError(f"arc carries {arc.n} observation sets for {n} filters")
        if len(arc) < 2:
            raise ODError("TooFewMeasurements: need 2")  # process/mod.rs:139-145
        from .cosmic import pack_spacecraft

        frame = initial_estimates[0].nominal_state.orbit.frame
        st, cs, ep = pack_spacecraft(e.nominal_state for e in initial_estimates)
        cov0 = np.empty((81, n))
        for i, e in enumerate(initial_estimates):
            cov0[:, i] = np.asarray(e.covar, dtype=np.float64).reshape(9, 9).T.reshape(81)  # (c*9 + r)
        eng = self.prop.engine(frame, self.almanac)
        if self.is_position:
            if not arc.is_position:
                raise ODError("position devices need a tracking arc of types (X, Y, Z)")
            names, dev_c = self.position_devices_c()
            tracker = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
            res = eng.od_position_batch(self.config_c(), len(names), dev_c, arc.epoch_ns, tracker, arc.obs, st, cs, ep, cov0,
                                        record_estimates=record_estimates, estimates_capacity=estimates_capacity)
        elif self.is_interlink:
            if self.msr_size == 3:
                raise ODError("msr_size 3 needs position devices")
            if tuple(arc.types) != (MeasurementType.Range, MeasurementType.Doppler):
                raise ODError("interlink devices need a tracking arc of types (Range, Doppler)")
            names, dev_c, sink = self.interlink_c(frame)
            tracker = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
            res = eng.od_interlink_batch(self.config_c(), len(names), dev_c, sink, arc.epoch_ns, tracker, arc.obs, st, cs, ep, cov0,
                                         record_estimates=record_estimates, estimates_capacity=estimates_capacity)
        else:
            if self.msr_size == 3:
                raise ODError("msr_size 3 needs position devices")
            if arc.is_position:
                raise ODError("ground stations need a tracking arc of types (Range, Doppler)")
            if arc.is_aer:
                names, st_c = self.aer_stations_c(frame)
                tracker = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
                res = eng.od_aer_batch(self.config_c(), len(names), st_c, arc.epoch_ns, tracker, arc.obs, st, cs, ep, cov0,
                                       record_estimates=record_estimates, estimates_capacity=estimates_capacity)
            else:
                if any(d.has_angles for d in self.devices.values()):
                    raise ODError("stations that measure azimuth or elevation need a tracking arc of types AER_TYPES")
                names, st_c = self.stations_c(frame)
                tracker = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
                rec_kw = {} if estimates_capacity is None else {"estimates_capacity": estimates_capacity}
                res = eng.od_ekf_batch(self.config_c(), len(names), st_c, arc.epoch_ns, tracker, arc.obs, st, cs, ep, cov0,
                                       record_estimates=record_estimates, **rec_kw)
        res.templates = [e.nominal_state for e in initial_estimates]
        res.arc = arc
        res.devices = self.devices
        res.process = self
        res.initial_estimates = list(initial_estimates)
        return res

    def process_arc(self, initial_estimate: KfEstimate, arc: TrackingDataArc) -> ODSolution:
        return self.process_arcs([initial_estimate], arc)

    # ---- covariance mapping (od/process/mod.rs:440-496)
    def predict_ensemble_until(self, estimates: Sequence[KfEstimate], end_epoch, capacity: Optional[int] = None,
                               record_states: bool = True, record_covars: bool = True) -> PredictionSolution:
        """n independent `predict_until(estimate_i, end_epoch_i)` runs in one launch; `end_epoch` is one epoch (ns) or one per
        estimate.  Each run starts from its estimate's nominal state, covariance and state deviation (so a CKF
        `ODSolution.final_estimate(i)` is predicted onward with its deviation).  `capacity` records are kept per run (default: as many
        as the longest run produces; 0 keeps the final estimates only)."""
        from .cosmic import pack_spacecraft

        n = len(estimates)
        if n == 0:
            raise ODError("no estimate to predict")
        cfg = self.config_c()
        frame = estimates[0].nominal_state.orbit.frame
        st, cs, ep = pack_spacecraft(e.nominal_state for e in estimates)
        end = np.ascontiguousarray(np.broadcast_to(np.asarray(end_epoch, dtype=np.int64), (n,)))
        if capacity is None:
            span = np.maximum(end - ep, 1)
            capacity = int(1 + ((span + cfg.max_step_ns - 1) // cfg.max_step_ns).max())
        cov0 = np.empty((81, n))
        dev0 = np.empty((9, n))
        for i, e in enumerate(estimates):
            cov0[:, i] = np.asarray(e.covar, dtype=np.float64).reshape(9, 9).T.reshape(81)  # (c*9 + r)
            dev0[:, i] = np.asarray(e.state_deviation, dtype=np.float64)
        eng = self.prop.engine(frame, self.almanac)
        res = eng.od_predict_batch(cfg, st, cs, ep, end, cov0, dev0, capacity=capacity, record_states=record_states,
                                   record_covars=record_covars)
        res.templates = [e.nominal_state for e in estimates]
        return res

    def predict_ensemble_for(self, estimates: Sequence[KfEstimate], duration: int, **kw) -> PredictionSolution:
        """`predict_ensemble_until` with end_i = epoch0_i + duration."""
        end = np.array([e.nominal_state.epoch() for e in estimates], dtype=np.int64) + int(duration)
        return self.predict_ensemble_until(estimates, end, **kw)

    def predict_until(self, initial_estimate: KfEstimate, end_epoch: int, **kw) -> PredictionSolution:
        """`KalmanODProcess::predict_until` (od/process/mod.rs:440-486)."""
        return self.predict_ensemble_until([initial_estimate], int(end_epoch), **kw)

    def predict_for(self, initial_estimate: KfEstimate, duration: int, **kw) -> PredictionSolution:
        """`KalmanODProcess::predict_for` (od/process/mod.rs:489-496)."""
        return self.predict_ensemble_for([initial_estimate], duration, **kw)


def SpacecraftKalmanOD(prop, kf_variant, sigma_reject, devices, almanac) -> KalmanODProcess:
    return KalmanODProcess(prop, kf_variant, sigma_reject, devices, almanac, msr_size=2)


def SpacecraftKalmanScalarOD(prop, kf_variant, sigma_reject, devices, almanac) -> KalmanODProcess:
    return KalmanODProcess(prop, kf_variant, sigma_reject, devices, almanac, msr_size=1)


class BLSSolver(enum.IntEnum):
    NormalEquations = abi.BLS_NORMAL_EQUATIONS
    LevenbergMarquardt = abi.BLS_LEVENBERG_MARQUARDT


_BLS_ERRORS = {abi.ERR_TOO_FEW_MEASUREMENTS: "TooFewMeasurements", abi.ERR_SINGULAR_INFORMATION: "SingularInformationMatrix",
               abi.ERR_INVALID_MEASUREMENT: "InvalidMeasurement"}


def _bls_error(status: int) -> Optional[str]:
    """The ODError a non-zero per-problem status stands for (propagation errors keep their status number)."""
    code = int(status) & 0xFF
    if code == 0:
        return None
    return _BLS_ERRORS.get(code, f"ODPropError (status {code})")


@dataclass
class BLSSolution:
    """`BLSSolution` (od/blse/solution.rs) of one problem."""

    estimated_state: Spacecraft
    covariance: np.ndarray           # [9][9]
    num_iterations: int
    final_rms: float
    final_corr_pos_km: float
    converged: bool

    def to_kf_estimate(self) -> KfEstimate:
        """`From<BLSSolution> for KfEstimate` (od/blse/solution.rs:75-93): the covariance with entries (6,6), (7,7) and (8,8) zeroed."""
        cov = np.array(self.covariance, dtype=np.float64).copy()
        for q in (6, 7, 8):
            cov[q, q] = 0.0
        return KfEstimate(self.estimated_state, cov)


@dataclass
class BLSEnsembleSolution:
    """Results of n batch least-squares problems solved in one launch; `solution(i)` is problem i's `BLSSolution`, `status[i]` its
    error (0: Ok; see `ODError` for the single-problem calls)."""

    state_soa: np.ndarray            # [9][n]
    epoch_ns: np.ndarray             # [n]
    covar: np.ndarray                # [n][9][9]
    iterations: np.ndarray           # [n]
    final_rms: np.ndarray            # [n]
    final_corr_pos_km: np.ndarray    # [n]
    converged: np.ndarray            # [n] bool
    details: np.ndarray
    status: np.ndarray
    templates: Sequence[Spacecraft] = ()

    def __len__(self):
        return self.status.shape[0]

    def error(self, i: int) -> Optional[str]:
        return _bls_error(self.status[i])

    def solution(self, i: int) -> BLSSolution:
        err = self.error(i)
        if err is not None:
            raise ODError(f"{err} (problem {i})")
        sc = self.templates[i].with_vector(int(self.epoch_ns[i]), self.state_soa[:, i])
        return BLSSolution(sc, self.covar[i].copy(), int(self.iterations[i]), float(self.final_rms[i]), float(self.final_corr_pos_km[i]),
                           bool(self.converged[i]))


class BatchLeastSquares:
    """`BatchLeastSquares<SpacecraftDynamics, GroundStation>` (od/blse/mod.rs:30-541) on the batched GPU path, with the reference's
    builder defaults (od/blse/mod.rs:80-135).  Every problem of an ensemble shares the devices and the schedule of
    the arc; each has its own initial guess and observation set."""

    def __init__(self, prop, devices: Dict[str, GroundStation], almanac: Optional[Almanac], solver: BLSSolver = BLSSolver.NormalEquations,
                 tolerance_pos_km: float = 1e-4, max_iterations: int = 10, max_step: int = 30 * NS_PER_S, epoch_precision: int = 1_000,
                 lm_lambda_init: float = 10.0, lm_lambda_decrease: float = 10.0, lm_lambda_increase: float = 10.0,
                 lm_lambda_min: float = 1e-12, lm_lambda_max: float = 1e12, lm_use_diag_scaling: bool = True):
        if any(isinstance(d, PositionDevice) for d in devices.values()):
            raise ODError("batch least squares takes ground stations only")
        if any(isinstance(d, InterlinkTxSpacecraft) for d in devices.values()):
            raise ODError("batch least squares does not take interlink devices on the GPU path")
        if any(d.has_angles for d in devices.values()):
            raise ODError("batch least squares takes range and Doppler only, not azimuth or elevation")
        self.prop = prop
        self.devices = dict(devices)
        self.almanac = almanac
        self.solver = BLSSolver(solver)
        self.tolerance_pos_km = float(tolerance_pos_km)
        self.max_iterations = int(max_iterations)
        self.max_step = int(max_step)
        self.epoch_precision = int(epoch_precision)
        self.lm_lambda_init = float(lm_lambda_init)
        self.lm_lambda_decrease = float(lm_lambda_decrease)
        self.lm_lambda_increase = float(lm_lambda_increase)
        self.lm_lambda_min = float(lm_lambda_min)
        self.lm_lambda_max = float(lm_lambda_max)
        self.lm_use_diag_scaling = bool(lm_use_diag_scaling)

    def config_c(self) -> abi.BlsConfigC:
        c = abi.BlsConfigC()
        c.solver = int(self.solver)
        c.max_iterations = self.max_iterations
        c.tolerance_pos_km = self.tolerance_pos_km
        c.max_step_ns = self.max_step
        c.epoch_precision_ns = self.epoch_precision
        c.lm_lambda_init, c.lm_lambda_decrease, c.lm_lambda_increase = self.lm_lambda_init, self.lm_lambda_decrease, self.lm_lambda_increase
        c.lm_lambda_min, c.lm_lambda_max = self.lm_lambda_min, self.lm_lambda_max
        c.lm_use_diag_scaling = int(self.lm_use_diag_scaling)
        return c

    def _pack(self, guesses: Sequence[Spacecraft], arc: TrackingDataArc):
        from .cosmic import pack_spacecraft

        n = len(guesses)
        if n == 0:
            raise ODError("no initial guess")
        if arc.n != n:
            raise ODError(f"arc carries {arc.n} observation sets for {n} problems")
        if arc.is_aer:
            raise ODError("batch least squares takes arcs of types (Range, Doppler), not AER_TYPES")
        frame = guesses[0].orbit.frame
        st, cs, ep = pack_spacecraft(guesses)
        eng = self.prop.engine(frame, self.almanac)
        names = list(self.devices)
        st_c = (abi.GroundStationC * max(len(names), 1))()
        for i, nme in enumerate(names):
            st_c[i] = self.devices[nme].to_c(frame, self.almanac)
        tracker = np.array([names.index(t) if t in names else -1 for t in arc.tracker], dtype=np.int32)
        return eng, (self.config_c(), len(names), st_c, arc.epoch_ns, tracker, arc.obs, st, cs, ep)

    def estimate_ensemble(self, guesses: Sequence[Spacecraft], arc: TrackingDataArc) -> BLSEnsembleSolution:
        """n independent `estimate(guess_i, arc_i)` runs in one launch; failures are per-problem statuses."""
        guesses = list(guesses)
        eng, args = self._pack(guesses, arc)
        r = eng.od_bls_batch(*args)
        return BLSEnsembleSolution(r["state"], r["epoch"], r["covar"], r["iterations"], r["final_rms"], r["final_corr_pos_km"],
                                   r["converged"] != 0, r["details"], r["status"], guesses)

    def estimate(self, initial_guess: Spacecraft, arc: TrackingDataArc) -> BLSSolution:
        """`BatchLeastSquares::estimate` (od/blse/mod.rs:146-446); raises ODError where the reference returns Err."""
        return self.estimate_ensemble([initial_guess], arc).solution(0)

    def evaluate_ensemble(self, states: Sequence[Spacecraft], arc: TrackingDataArc):
        """n independent `evaluate(state_i, arc_i)` runs in one launch: (rms[n], status[n])."""
        eng, args = self._pack(list(states), arc)
        return eng.od_bls_evaluate_batch(*args)

    def evaluate(self, state: Spacecraft, arc: TrackingDataArc) -> float:
        """`BatchLeastSquares::evaluate` (od/blse/mod.rs:450-541): the RMS of the weighted residuals of `state` over the arc."""
        rms, status = self.evaluate_ensemble([state], arc)
        err = _bls_error(status[0])
        if err is not None:
            raise ODError(err)
        return float(rms[0])


# --------------------------------------------------------------------------- measurement simulation (host-side data generation)
def _rotation_matrix(rot, t_ns: int) -> np.ndarray:
    """inertial -> body-fixed DCM of the orientation model of include/nyxb.h (numpy restatement for the simulator)."""
    if rot is None or rot.kind == 0:
        return np.eye(3)
    d = duration_to_seconds(int(t_ns)) / 86400.0
    T = d / 36525.0
    ra = math.radians(rot.ra0_deg + rot.ra1_deg_cy * T)
    dec = math.radians(rot.dec0_deg + rot.dec1_deg_cy * T)
    w = math.radians(math.fmod(rot.w0_deg + rot.w1_deg_day * d, 360.0))
    sa, ca, sd, cd, sw, cw = math.sin(ra), math.cos(ra), math.sin(dec), math.cos(dec), math.sin(w), math.cos(w)
    ba = np.array([[-sa, ca, 0.0], [-sd * ca, -sd * sa, cd], [cd * ca, cd * sa, sd]])
    r3 = np.array([[cw, sw, 0.0], [-sw, cw, 0.0], [0.0, 0.0, 1.0]])
    return r3 @ ba


def station_state(gs: GroundStation, t_ns: int, integration_frame: Frame, almanac: Optional[Almanac]):
    """Inertial position/velocity of the antenna relative to the integration centre (trk_device.rs:150-152)."""
    pos_f, up = gs.body_fixed()
    R = _rotation_matrix(gs.frame.rotation, t_ns)
    wdot = math.radians(gs.frame.rotation.w1_deg_day) / 86400.0 if gs.frame.rotation is not None and gs.frame.rotation.kind else 0.0
    r = R.T @ pos_f
    v = R.T @ np.cross(np.array([0.0, 0.0, wdot]), pos_f)
    if gs.frame.ephemeris_id != integration_frame.ephemeris_id:
        b = almanac.bodies[almanac.body_index(gs.frame.ephemeris_id)]
        dt = 1_000_000_000
        p0 = b.position(t_ns)
        vb = (b.position(t_ns + dt) - b.position(t_ns - dt)) / (2.0 * dt / NS_PER_S)
        r, v = r + p0, v + vb
    return r, v, R.T @ up


def simulate_tracking(truth_epochs_ns, truth_states, devices: Dict[str, GroundStation], schedule: Sequence[str], frame: Frame,
                      almanac: Optional[Almanac], rng: Optional[np.random.Generator] = None) -> TrackingDataArc:
    """Synthetic range / Doppler observations of `truth_states[k]` ([m][6][n]) at `truth_epochs_ns[k]` from tracker
    `schedule[k]`; white noise of each station's sigma when `rng` is given.  Invisible passes are NaN (absent).  When a station
    carries azimuth or elevation the arc has types AER_TYPES (obs [m][4][n]) and the angles, in degrees, are those of
    nyxb_aer_station (azimuth in [0, 360) before noise)."""
    truth_states = np.asarray(truth_states, dtype=np.float64)
    m, _, n = truth_states.shape
    aer = any(gs.has_angles for gs in devices.values())
    obs = np.full((m, 4 if aer else 2, n), np.nan)
    for k in range(m):
        gs = devices[schedule[k]]
        r_tx, v_tx, up_in = station_state(gs, int(truth_epochs_ns[k]), frame, almanac)
        rho = truth_states[k, :3, :] - r_tx[:, None]
        dv = truth_states[k, 3:6, :] - v_tx[:, None]
        rng_km = np.linalg.norm(rho, axis=0)
        rr = (rho * dv).sum(0) / rng_km
        elev = np.degrees(np.arcsin((rho * up_in[:, None]).sum(0) / rng_km))
        if aer:
            R = _rotation_matrix(gs.frame.rotation, int(truth_epochs_ns[k]))
            north, east = (R.T @ u for u in gs.north_east_fixed())
            az = np.mod(np.degrees(np.arctan2((rho * east[:, None]).sum(0), (rho * north[:, None]).sum(0))), 360.0)
        vis = elev >= gs.elevation_mask_deg
        if gs.frame.ephemeris_id != frame.ephemeris_id:
            # line of sight blocked by the body the spacecraft orbits (Vallado's SIGHT)
            r1, r2 = truth_states[k, :3, :], r_tx[:, None] * np.ones((1, n))
            r1sq, r2sq, r12 = (r1 * r1).sum(0), (r2 * r2).sum(0), (r1 * r2).sum(0)
            tau = (r1sq - r12) / (r1sq + r2sq - 2.0 * r12)
            blocked = (tau >= 0.0) & (tau <= 1.0) & ((1.0 - tau) * r1sq + r12 * tau <= frame.mean_equatorial_radius_km() ** 2)
            vis &= ~blocked
        for t in gs.measurement_types:
            val = {MeasurementType.Range: rng_km, MeasurementType.Doppler: rr}.get(t)
            if val is None:
                val = az if t == MeasurementType.Azimuth else elev
            noise = rng.normal(0.0, gs.stochastic_noises[t].sigma, n) if rng is not None else 0.0
            obs[k, int(t), :] = np.where(vis, val + noise, np.nan)
    return TrackingDataArc(np.asarray(truth_epochs_ns, dtype=np.int64), list(schedule), obs,
                           AER_TYPES if aer else (MeasurementType.Range, MeasurementType.Doppler))


def simulate_position_fixes(truth_epochs_ns, truth_states, devices: Dict[str, PositionDevice], schedule: Sequence[str],
                            rng: Optional[np.random.Generator] = None) -> TrackingDataArc:
    """Synthetic position fixes of `truth_states[k]` ([m][>=3][n], integration frame) at `truth_epochs_ns[k]` from device
    `schedule[k]`, as `measure_instantaneous` with an RNG (position/trk_device.rs:76-83): the value of the type at list position ii is
    position component ii, plus white noise of the type's sigma when `rng` is given, plus the type's constant bias.  Returns an arc of
    types (X, Y, Z); the types a device does not carry are NaN."""
    truth_states = np.asarray(truth_states, dtype=np.float64)
    m, _, n = truth_states.shape
    obs = np.full((m, 3, n), np.nan)
    for k in range(m):
        dev = devices[schedule[k]]
        for ii, t in enumerate(dev.measurement_types):
            nz = dev.stochastic_noises[t]
            noise = rng.normal(0.0, nz.sigma, n) if rng is not None else 0.0
            obs[k, int(t) - abi.MSR_X, :] = (truth_states[k, ii, :] + noise) + nz.bias_constant
    return TrackingDataArc(np.asarray(truth_epochs_ns, dtype=np.int64), list(schedule), obs, _POSITION_TYPES)


def interlink_geometry(tx_rv, rx_rv):
    """(range, range rate) of the receiver states rx_rv ([6][n]) seen from the transmitter states tx_rv ([6][n]) as the reference
    computes them (interlink/trk_device.rs:195-210): rho = r_rx - r_tx and rho . v_rx / |rho|, the transmitter's velocity left out."""
    rho = rx_rv[:3] - tx_rv[:3]
    rng_km = np.sqrt((rho[0] * rho[0] + rho[1] * rho[1]) + rho[2] * rho[2])
    return rng_km, ((rho[0] * rx_rv[3] + rho[1] * rx_rv[4]) + rho[2] * rx_rv[5]) / rng_km


def simulate_interlink(truth_epochs_ns, truth_states, devices: Dict[str, InterlinkTxSpacecraft], schedule: Sequence[str], frame: Frame,
                       rng: Optional[np.random.Generator] = None) -> TrackingDataArc:
    """Synthetic interlink observations of the receivers `truth_states[k]` ([m][6][n], integration frame) at `truth_epochs_ns[k]`
    from transmitter `schedule[k]`, with the reference simulator's geometry (measure_instantaneous, interlink/trk_device.rs:180-232):
    the transmitter is `traj.at(epoch)`, the link is blocked by the body at the frame's centre (Vallado's SIGHT), and the Doppler
    ignores the transmitter's velocity, so these data agree with the filter's computed observation.  White noise of each type's sigma
    and the constant bias when `rng` is given.  Blocked links are NaN (absent).  Returns a (Range, Doppler) arc.  Host-side test data,
    not a GPU simulator."""
    truth_states = np.asarray(truth_states, dtype=np.float64)
    m, _, n = truth_states.shape
    radius = frame.mean_equatorial_radius_km()
    obs = np.full((m, 2, n), np.nan)
    for k in range(m):
        dev = devices[schedule[k]]
        tx = dev.traj.at(int(truth_epochs_ns[k])).orbit.to_cartesian_pos_vel()
        r1 = truth_states[k, :3, :]                          # receiver first, as the ground station's test
        r2 = np.asarray(tx[:3], dtype=np.float64)[:, None] * np.ones((1, n))
        r1sq, r2sq, r12 = (r1[0] * r1[0] + r1[1] * r1[1]) + r1[2] * r1[2], (r2[0] * r2[0] + r2[1] * r2[1]) + r2[2] * r2[2], \
            (r1[0] * r2[0] + r1[1] * r2[1]) + r1[2] * r2[2]
        tau = (r1sq - r12) / (r1sq + r2sq - 2.0 * r12)
        blocked = (tau >= 0.0) & (tau <= 1.0) & ((1.0 - tau) * r1sq + r12 * tau <= radius * radius)
        rng_km, rr = interlink_geometry(np.asarray(tx, dtype=np.float64)[:, None] * np.ones((1, n)), truth_states[k, :6, :])
        for t in dev.measurement_types:
            t = MeasurementType(t)
            nz = dev.stochastic_noises[t]
            noise = rng.normal(0.0, nz.sigma, n) + nz.bias_constant if rng is not None else 0.0
            obs[k, int(t), :] = np.where(blocked, np.nan, (rng_km if t == MeasurementType.Range else rr) + noise)
    return TrackingDataArc(np.asarray(truth_epochs_ns, dtype=np.int64), list(schedule), obs)
