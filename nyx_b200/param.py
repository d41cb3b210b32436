"""`StateParameter` (md/param.rs:34-70) and `Spacecraft::value` (cosmic/spacecraft.rs:520-578), vectorised over arrays of states.

The reference's `StateParameter::Element(e)` wraps anise's `OrbitalElement` (not in the reference tree) and evaluates it through
`e.evaluate(orbit)`; the elements offered here are the ones the path's consumers name — `Spacecraft::export_params`
(md/trajectory/interpolatable.rs:118-147), the Monte Carlo reports (mc/results.rs:88-240), the dispersions
(mc/multivariate.rs:80-178) — computed with the textbook two-body relations (parity unpinned at the anise boundary; angles in
degrees in [0, 360), like anise's).  Parameters that need a thruster or a guidance law (Isp, Thrust, ThrustX.., GuidanceMode,
B-plane) are `StateError::Unavailable` on this path: the engine integrates unguided spacecraft (SURVEY.md §8 a9).
"""
from __future__ import annotations

import enum

import numpy as np


class StateError(RuntimeError):
    """`StateError::Unavailable { param }` / `NoThrusterAvail` (errors.rs)."""


class StateParameter(enum.Enum):
    # Element(OrbitalElement::..)
    X = "X (km)"
    Y = "Y (km)"
    Z = "Z (km)"
    VX = "VX (km/s)"
    VY = "VY (km/s)"
    VZ = "VZ (km/s)"
    Rmag = "Rmag (km)"
    Vmag = "Vmag (km/s)"
    SemiMajorAxis = "SemiMajorAxis (km)"
    Eccentricity = "Eccentricity"
    Inclination = "Inclination (deg)"
    RAAN = "RAAN (deg)"
    AoP = "AoP (deg)"
    TrueAnomaly = "TrueAnomaly (deg)"
    AoL = "AoL (deg)"
    TrueLongitude = "TrueLongitude (deg)"
    Period = "Period (s)"
    Energy = "Energy (km^2/s^2)"
    Hmag = "Hmag (km^2/s)"
    ApoapsisRadius = "ApoapsisRadius (km)"
    PeriapsisRadius = "PeriapsisRadius (km)"
    C3 = "C3 (km^2/s^2)"
    Declination = "Declination (deg)"
    # md/param.rs:172-196 Display names
    Cd = "cd"
    Cr = "cr"
    DryMass = "dry_mass (kg)"
    PropMass = "prop_mass (kg)"
    TotalMass = "total_mass (kg)"
    Isp = "isp (isp)"
    Thrust = "thrust (N)"
    GuidanceMode = "guidance_mode"

    def __str__(self) -> str:
        return self.value

    @property
    def unit(self) -> str:
        name = self.value
        return name[name.index("(") + 1:-1] if "(" in name else ""


#: `Spacecraft::export_params` (interpolatable.rs:118-147) minus the thruster/guidance entries, which are all-null on this path
#: and therefore dropped by `to_parquet` (mc/results.rs:326-343: a field no state can evaluate is not written)
EXPORT_PARAMS = [StateParameter.X, StateParameter.Y, StateParameter.Z, StateParameter.VX, StateParameter.VY, StateParameter.VZ,
                 StateParameter.SemiMajorAxis, StateParameter.Eccentricity, StateParameter.Inclination, StateParameter.RAAN,
                 StateParameter.AoP, StateParameter.TrueAnomaly, StateParameter.AoL, StateParameter.TrueLongitude,
                 StateParameter.DryMass, StateParameter.PropMass, StateParameter.Cr, StateParameter.Cd]

_UNAVAILABLE = (StateParameter.Isp, StateParameter.Thrust, StateParameter.GuidanceMode)
_CART = {StateParameter.X: 0, StateParameter.Y: 1, StateParameter.Z: 2, StateParameter.VX: 3, StateParameter.VY: 4, StateParameter.VZ: 5}


def _wrap360(a):
    a = np.mod(a, 360.0)
    return np.where(a < 0.0, a + 360.0, a)


def _angle(cosv, flip):
    ang = np.degrees(np.arccos(np.clip(cosv, -1.0, 1.0)))
    return np.where(flip, 360.0 - ang, ang)


def evaluate(param: StateParameter, rv: np.ndarray, mu_km3_s2: float, template=None, cr=None, cd=None, prop_mass_kg=None):
    """Values of `param` for the Cartesian states rv[6, ...] (km, km/s) around a body of gravitational parameter mu.
    `template` supplies the masses and coefficients that stay constant on this path; `cr`, `cd`, `prop_mass_kg` override them
    per state (the dispersed values of a Monte Carlo run).  Raises StateError for parameters unavailable on this path."""
    if not isinstance(param, StateParameter):
        raise StateError(f"unknown state parameter {param!r}")
    if param in _UNAVAILABLE:
        raise StateError(f"{param} unavailable: no thruster / guidance on the propagation path")
    rv = np.asarray(rv, dtype=np.float64)
    shape = rv.shape[1:]
    if param in _CART:
        return rv[_CART[param]].copy()

    def const(override, attr):
        if override is not None:
            return np.broadcast_to(np.asarray(override, dtype=np.float64), shape).copy()
        if template is None:
            raise StateError(f"{param} needs a spacecraft template")
        return np.full(shape, attr(template))

    if param is StateParameter.Cr:
        return const(cr, lambda t: t.srp.coeff_reflectivity)
    if param is StateParameter.Cd:
        return const(cd, lambda t: t.drag.coeff_drag)
    if param is StateParameter.DryMass:
        return const(None, lambda t: t.mass.dry_mass_kg)
    if param is StateParameter.PropMass:
        return const(prop_mass_kg, lambda t: t.mass.prop_mass_kg)
    if param is StateParameter.TotalMass:
        return const(None, lambda t: t.mass.dry_mass_kg + t.mass.extra_mass_kg) + const(prop_mass_kg, lambda t: t.mass.prop_mass_kg)

    r, v = rv[:3], rv[3:]
    rmag = np.sqrt((r * r).sum(axis=0))
    vmag = np.sqrt((v * v).sum(axis=0))
    if param is StateParameter.Rmag:
        return rmag
    if param is StateParameter.Vmag:
        return vmag
    if param is StateParameter.Declination:
        return np.degrees(np.arcsin(r[2] / rmag))
    energy = 0.5 * vmag * vmag - mu_km3_s2 / rmag
    if param is StateParameter.Energy:
        return energy
    sma = -mu_km3_s2 / (2.0 * energy)
    if param is StateParameter.SemiMajorAxis:
        return sma
    if param is StateParameter.C3:
        return -mu_km3_s2 / sma
    if param is StateParameter.Period:
        return 2.0 * np.pi * np.sqrt(sma * sma * sma / mu_km3_s2)
    h = np.cross(r, v, axis=0)
    hmag = np.sqrt((h * h).sum(axis=0))
    if param is StateParameter.Hmag:
        return hmag
    rdv = (r * v).sum(axis=0)
    evec = ((vmag * vmag - mu_km3_s2 / rmag) * r - rdv * v) / mu_km3_s2
    ecc = np.sqrt((evec * evec).sum(axis=0))
    if param is StateParameter.Eccentricity:
        return ecc
    if param is StateParameter.ApoapsisRadius:
        return sma * (1.0 + ecc)
    if param is StateParameter.PeriapsisRadius:
        return sma * (1.0 - ecc)
    if param is StateParameter.Inclination:
        return np.degrees(np.arccos(np.clip(h[2] / hmag, -1.0, 1.0)))
    node = np.stack([-h[1], h[0], np.zeros_like(hmag)])   # z x h
    nmag = np.sqrt((node * node).sum(axis=0))
    with np.errstate(invalid="ignore", divide="ignore"):
        raan = _angle(node[0] / nmag, node[1] < 0.0)
        aop = _angle((node * evec).sum(axis=0) / (nmag * ecc), evec[2] < 0.0)
        ta = _angle((evec * r).sum(axis=0) / (ecc * rmag), rdv < 0.0)
    if param is StateParameter.RAAN:
        return raan
    if param is StateParameter.AoP:
        return aop
    if param is StateParameter.TrueAnomaly:
        return ta
    if param is StateParameter.AoL:
        return _wrap360(aop + ta)
    if param is StateParameter.TrueLongitude:
        return _wrap360(aop + raan + ta)
    raise StateError(f"{param} unavailable")
