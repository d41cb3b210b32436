"""nyx_b200 — H100-native (sm_90a) batched orbit propagation behind the nyx `Propagator` / `MonteCarlo` surface.

The package holds only what the hot path needs: ``csrc/`` (CUDA kernels + the C ABI declared in
``include/nyxb.h``) and a host-side mirror of the reference interface for that path.
There is NO CPU fallback: every propagate call goes through ``libnyxb.so`` on a CUDA device.
"""
from . import abi
from .abi import KERNEL_AUTO, KERNEL_COOP, KERNEL_THREAD, KERNEL_TRANSPOSED, MODE_FAST, MODE_STRICT, NyxbLibraryMissing
from .cosmic import DragData, Mass, Orbit, Spacecraft, SRPData, Unit, duration_to_seconds, epochs_to_utc_iso, pack_spacecraft, utc_iso_to_epochs
from .dynamics import (AtmDensity, Drag, DynamicsError, GravityField, OrbitalDynamics, PointMasses, ShadowModel,
                       SolarPressure, SpacecraftDynamics)
from .frames import (EARTH, EARTH_J2000, GMAT_EARTH_GM, GMAT_MOON_GM, GMAT_SUN_GM, IAU_EARTH_FRAME, IAU_MOON_FRAME,
                     JUPITER_BARYCENTER, JUPITER_BARYCENTER_J2000, MOON, MOON_J2000, SUN, SUN_J2000, Almanac, Frame,
                     Rotation)
from .gravity import GravityFieldData
from .monte_carlo import DispersedState, MonteCarlo, MonteCarloError, MvnSpacecraft, Results, Run, StateDispersion
from .param import EXPORT_PARAMS, StateError, StateParameter
from .trajectory import Traj, TrajError, hermite_eval
from . import dhall
from .config import PropagatorConfig, integrator_options_from, load_ground_stations, parse_duration
from .event import Event, brent, locate_event
from .od import (BatchLeastSquares, BLSEnsembleSolution, BLSSolution, BLSSolver, GroundStation, KalmanODProcess, KalmanVariant, KfEstimate, LocalFrame, MeasurementType, ODError, ODSolution,
                 PredictionSolution, ProcessNoise3D, SigmaRejection, SpacecraftKalmanOD, SpacecraftKalmanScalarOD, SpacecraftUncertainty,
                 StochasticNoise, TrackingDataArc, simulate_tracking, station_state)
from .od import AER_TYPES, InterlinkTxSpacecraft, PositionDevice, simulate_interlink, simulate_position_fixes
from .propagator import (Engine, ErrorControl, IntegrationDetails, IntegratorMethod, IntegratorOptions, PropagationError,
                         PropInstance, Propagator)
from .targeter import (Objective, Targeter, TargeterEnsembleSolution, TargeterSolution, TargetingError, Variable, Vary)

__all__ = [n for n in dir() if not n.startswith("_")]
