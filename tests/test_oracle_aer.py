"""The angle measurements of a ground station (nyxb_aer_station) on the CPU restatement (tests/aer_oracle.py): the reference's
sensitivity check, the sensitivity rows as coded, the angles against an independent SEZ arbiter, the mask, the azimuth wrap, the window
split and the ABI's argument checks."""
import ctypes as C
import math

import numpy as np

import nyx_b200 as nb
from nyx_b200 import abi
from nyx_b200.od import MeasurementType as MT
from tests import aer_oracle as ao
from tests import aer_util as au

R2D = 180.0 / math.pi


def _madrid(types=au.ALL, mask=0.0):
    return au.dsn(mask, types, names=("Madrid",))["Madrid"]


def _cislunar():
    """verif_sensitivity_mat's state (tests/orbit_determination/measurements.rs:334-404), Earth J2000."""
    t = int(nb.utc_iso_to_epochs(["2022-11-16T13:35:31"])[0])
    y = np.array([58643.769540, -61696.435624, -36178.745722, 2.148654, -1.202489, -0.714016, 0.0, 0.0, 0.0])
    return t, y


def _obs(g):
    return np.array([g["rng"], g["rr"], g["az"], g["elev"]])


def test_verif_sensitivity_mat_restated():
    """truth_obs - H (truth - pert) against pert_obs, for the four types, within the reference's 1e-3 bound.  The angles pass only
    because their true change is below 1e-3 deg: H's rad/km rows give H.delta about 180/pi too small."""
    t, y = _cislunar()
    yp = y + np.array([1.0, -1.0, 1.0, 1e-3, -1e-3, 1e-3, 0.0, 0.0, 0.0])
    gs = _madrid().to_aer_c(nb.EARTH_J2000, None)
    g, gp = ao.geometry(gs, None, t, y), ao.geometry(gs, None, t, yp)
    assert abs(g["elev"] - 7.4) < 0.1 and abs(g["az"] - 133.8) < 0.1 and abs(g["rng"] - 91442.0) < 1.0
    truth, pert = _obs(g), _obs(gp)
    errs = {}
    for t_ in (MT.Range, MT.Doppler, MT.Elevation, MT.Azimuth):
        H = np.array(ao.h_row(int(t_), g, truth))
        err = pert[int(t_)] - (truth[int(t_)] - H @ (y - yp))
        errs[t_] = err
        assert abs(err) < 1e-3, (t_, err)
    # the angle errors are nearly the whole true change: H.delta is tiny against it
    for t_ in (MT.Azimuth, MT.Elevation):
        H = np.array(ao.h_row(int(t_), g, truth))
        true_change = pert[int(t_)] - truth[int(t_)]
        assert abs(H @ (yp - y)) < 5e-2 * abs(true_change)
    assert 4e-4 < abs(errs[MT.Azimuth]) < 7e-4 and 6e-4 < abs(errs[MT.Elevation]) < 9e-4


def test_sensitivity_rows_as_coded():
    """Bit for bit: azimuth [-dy, dx, 0] / (dx^2 + dy^2); elevation with r^2 = (sqrt((dx^2 + dy^2) + dz^2))^2, which differs from the
    plain sum in the last bits for some inputs.  Neither row is the gradient of the computed angle: rad against deg, and the
    integration frame against SEZ."""
    rng = np.random.default_rng(3)
    differs = 0
    for _ in range(200):
        dr = rng.normal(0, 1e4, 3)
        g = dict(dr=list(dr), dv=[0.0] * 3, rng=0.0)
        az = ao.h_row(abi.MSR_AZIMUTH, g, None)
        el = ao.h_row(abi.MSR_ELEVATION, g, None)
        dx, dy, dz = dr
        den = dx * dx + dy * dy
        assert az[:3] == [-dy / den, dx / den, 0.0] and az[3:] == [0.0] * 6
        r2 = math.sqrt((dx * dx + dy * dy) + dz * dz) ** 2
        s = math.sqrt(r2 - dz * dz)
        assert el[:3] == [-(dx * dz) / (r2 * s), -(dy * dz) / (r2 * s), math.sqrt(dx * dx + dy * dy) / r2] and el[3:] == [0.0] * 6
        differs += r2 != (dx * dx + dy * dy) + dz * dz
    assert differs > 0
    # finite differences of the computed angles (deg/km) against the rows (rad/km, integration frame)
    t, y = _cislunar()
    gs = _madrid().to_aer_c(nb.EARTH_J2000, None)
    g = ao.geometry(gs, None, t, y)
    for typ, key in ((abi.MSR_AZIMUTH, "az"), (abi.MSR_ELEVATION, "elev")):
        fd = np.array([(ao.geometry(gs, None, t, y + h)[key] - ao.geometry(gs, None, t, y - h)[key]) / 2e-3
                       for h in np.eye(9)[:3] * 1e-3])
        H = np.array(ao.h_row(typ, g, _obs(g))[:3])
        assert np.linalg.norm(fd - H) > 0.5 * np.linalg.norm(fd)             # not the gradient
        assert np.linalg.norm(fd - R2D * H) > 1e-3 * np.linalg.norm(fd)      # nor after the unit change: the frame differs too


def _sez_arbiter(gs_model, t, y):
    """Independent arbiter: rho into the body-fixed frame, then into SEZ by rot2(90 deg - lat) . rot3(lon)."""
    gs_c = gs_model.to_aer_c(nb.EARTH_J2000, None)
    R = nb.od._rotation_matrix(gs_model.frame.rotation, t)
    pos, _ = gs_model.body_fixed()
    rho_bf = R @ y[:3] - pos
    lat, lon = math.radians(gs_model.latitude_deg), math.radians(gs_model.longitude_deg)

    def rot2(a):
        return np.array([[math.cos(a), 0.0, -math.sin(a)], [0.0, 1.0, 0.0], [math.sin(a), 0.0, math.cos(a)]])

    def rot3(a):
        return np.array([[math.cos(a), math.sin(a), 0.0], [-math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]])

    sez = rot2(math.pi / 2 - lat) @ rot3(lon) @ rho_bf
    az = math.degrees(math.atan2(sez[1], -sez[0])) % 360.0
    el = math.degrees(math.asin(sez[2] / np.linalg.norm(sez)))
    return gs_c, az, el


def test_angles_against_sez_arbiter():
    rng = np.random.default_rng(5)
    t0, _ = _cislunar()
    for nm in ("Madrid", "Canberra", "Goldstone"):
        model = au.dsn(0.0, names=(nm,))[nm]
        for _ in range(20):
            y = np.zeros(9)
            y[:3] = rng.normal(0, 3e4, 3)
            t = t0 + int(rng.integers(0, 86400)) * 10**9
            gs_c, az, el = _sez_arbiter(model, t, y)
            g = ao.geometry(gs_c, None, t, y)
            daz = (g["az"] - az + 180.0) % 360.0 - 180.0
            assert abs(daz) < 1e-12 and abs(g["elev"] - el) < 1e-12, (daz, g["elev"] - el)
            assert 0.0 <= g["az"] < 360.0


def test_observed_elevation_is_the_mask_elevation():
    """A mask equal to the computed elevation keeps the measurement; the next double above it hides it."""
    t, y = _cislunar()
    model = _madrid()
    gs = model.to_aer_c(nb.EARTH_J2000, None)
    el = ao.geometry(gs, None, t, y)["elev"]
    o = np.full(4, 1.0)
    gs.elevation_mask_deg = el
    w = ao.window(gs, None, 2, 1, o, t, y)
    assert not isinstance(w, str) and w[5][1] == el - gs.bias[3]
    gs.elevation_mask_deg = np.nextafter(el, np.inf)
    assert ao.window(gs, None, 2, 1, o, t, y) == "not_visible"


def test_azimuth_wrap_is_kept():
    """Nothing wraps the residual: an observed 359.99 deg against a computed azimuth near 0.01 deg is a prefit near 359.98 deg."""
    t, _ = _cislunar()
    model = _madrid(types=(MT.Azimuth,))
    gs = model.to_aer_c(nb.EARTH_J2000, None)
    R = nb.od._rotation_matrix(model.frame.rotation, t)
    pos, up = model.body_fixed()
    north, east = model.north_east_fixed()
    a = math.radians(0.01)
    y = np.zeros(9)
    y[:3] = R.T @ (pos + 1e4 * (math.cos(a) * north + math.sin(a) * east + 0.5 * up))
    w = ao.window(gs, None, 1, 0, np.array([np.nan, np.nan, 359.99, np.nan]), t, y)
    cur, avail, real, H, Rk, comp = w
    assert abs(comp[0] - 0.01) < 1e-6 and abs((real - comp)[0] - 359.98) < 1e-6
    y[:3] = R.T @ (pos + 1e4 * (math.cos(a) * north - math.sin(a) * east + 0.5 * up))
    w = ao.window(gs, None, 1, 0, np.array([np.nan, np.nan, 0.01, np.nan]), t, y)
    assert abs(w[5][0] - 359.99) < 1e-6 and abs((w[2] - w[5])[0] + 359.98) < 1e-6


def test_window_split_el_r_az():
    """[El, R, Az] at msr_size 2: windows [El, R] and [Az]; the short window keeps an identity row, a zero R entry and a zero real
    observation in its second slot.  At msr_size 1 three windows."""
    t, y = _cislunar()
    gs = _madrid(types=(MT.Elevation, MT.Range, MT.Azimuth)).to_aer_c(nb.EARTH_J2000, None)
    o = np.array([91442.0, 0.0, 133.8, 7.4])
    w0, w1 = ao.window(gs, None, 2, 0, o, t, y), ao.window(gs, None, 2, 1, o, t, y)
    assert w0[0] == [abi.MSR_ELEVATION, abi.MSR_RANGE] and list(w0[2]) == [7.4, 91442.0]
    assert list(w0[4]) == [gs.noise_var[0], gs.noise_var[1]]
    assert w1[0] == [abi.MSR_AZIMUTH] and w1[2][1] == 0.0 and w1[4][1] == 0.0 and list(w1[3][1]) == list(np.eye(9)[1])
    assert ao.window(gs, None, 2, 2, o, t, y) == "empty"
    assert [ao.window(gs, None, 1, w, o, t, y)[0] for w in range(3)] == [[3], [0], [2]]


def test_with_msr_type_builder():
    gs = nb.GroundStation.dss65_madrid(0.0, nb.StochasticNoise(1e-3), nb.StochasticNoise(1e-6))
    gs.with_msr_type(MT.Azimuth, nb.StochasticNoise(1e-2)).with_msr_type(MT.Range, nb.StochasticNoise(5e-3))
    assert list(gs.measurement_types) == [MT.Range, MT.Doppler, MT.Azimuth] and gs.stochastic_noises[MT.Range].sigma == 5e-3
    c = gs.to_aer_c(nb.EARTH_J2000, None)
    assert c.n_types == 3 and list(c.types) == [0, 1, 2, 0] and c.noise_var[2] == 1e-4
    north, east = gs.north_east_fixed()
    _, up = gs.body_fixed()
    assert abs(north @ east) < 1e-15 and abs(north @ up) < 1e-15 and np.allclose(np.cross(east, north), up, atol=1e-15)


def test_abi_struct_sizes_and_null_arguments():
    """The checks that need no engine.  The checks on types, duplicates, n_types and msr_size read the engine (its bodies and setup),
    and an engine cannot be created without a CUDA device (nyxb_engine_create refuses: no CPU fallback); they are pinned, with the
    engine's launch count unchanged by every rejected call, in tests/test_gpu_aer.py::test_argument_checks."""
    lib = abi.load_library()
    assert C.sizeof(abi.AerStationC) == 256 and C.sizeof(abi.GroundStationC) == 176
    assert lib.nyxb_od_aer_batch(None, None, 0, None, None, 1, None, None, None, None, None, None) == -1
    assert b"null" in lib.nyxb_last_error()
    assert lib.nyxb_od_aer_smooth_batch(None, None, 0, None, None, 1, None, None, None) == -1
    assert b"null" in lib.nyxb_last_error()
