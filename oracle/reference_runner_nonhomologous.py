"""Run the UNMODIFIED reference's nonhomologous Monte Carlo loop on a synthetic model.

TEST INFRASTRUCTURE ONLY (see oracle/reference_loader.py).  `montecarlo_transport_with_vpackets`
(tardis/transport/montecarlo/modes/montecarlo_transport.py:239) with the nonhomologous `packet_propagation`
(modes/nonhomologous/packet_propagation.py:53) and NumbaRadial1DGeometry, called with time_explosion = 0.0 as
MCTransportSolverNonhomologous.run does (modes/nonhomologous/solver.py:213-229).
"""
from __future__ import annotations

import numpy as np

from . import reference_loader
from .reference_runner import build_reference_objects


def load():
    R = reference_loader.load()
    from tardis.model.geometry.radial1d import NumbaRadial1DGeometry
    from tardis.transport.geometry.calculate_distances import calculate_distance_line_nonhomologous
    from tardis.transport.montecarlo.modes.nonhomologous.packet_propagation import packet_propagation
    from tardis.transport.montecarlo.nonhomologous_grid import depressed_quartic
    from tardis.transport.montecarlo.packets.radiative_packet import RPacket

    R.NumbaRadial1DGeometry = NumbaRadial1DGeometry
    R.calculate_distance_line_nonhomologous = calculate_distance_line_nonhomologous
    R.nonhomologous_packet_propagation = packet_propagation
    R.depressed_quartic = depressed_quartic
    R.RPacket = RPacket
    return R


def geometry(model):
    return load().NumbaRadial1DGeometry(model.r_inner.copy(), model.r_outer.copy(), model.v_inner.copy(), model.v_outer.copy())


def run_reference_nonhomologous(model, packets, *, number_of_vpackets=0, disable_line_scattering=False,
                                survival_probability=0.0, track_full=False, nthreads=1):
    """One reference MC iteration of the nonhomologous mode: dict of numpy outputs (as oracle.reference_runner)."""
    import numba

    R = load()
    _, _, opacity, cfg, pc = build_reference_objects(
        model, packets, number_of_vpackets=number_of_vpackets, disable_line_scattering=disable_line_scattering,
        survival_probability=survival_probability)
    geo = geometry(model)
    numba.set_num_threads(nthreads)
    n = len(packets)
    trackers = R.generate_tracker_full_list(n, 10) if track_full else R.generate_tracker_last_interaction_list(n)
    vhist, _, bulk, line = R.montecarlo_transport_with_vpackets(
        pc, geo, 0.0, opacity, cfg, model.spectrum_frequency_grid, trackers, number_of_vpackets, False,
        R.nonhomologous_packet_propagation)
    out = dict(
        output_nus=np.asarray(pc.output_nus).copy(), output_energies=np.asarray(pc.output_energies).copy(),
        j=np.asarray(bulk.mean_intensity_total).copy(), nu_bar=np.asarray(bulk.mean_frequency).copy(),
        j_blue=np.asarray(line.mean_intensity_blueward).copy(), edotlu=np.asarray(line.energy_deposition_line_rate).copy(),
        vhist=np.asarray(vhist).copy(), velocity_gradient=np.asarray(geo.velocity_gradient).copy(),
    )
    out["last_interaction_type"] = np.array([t.interaction_type for t in trackers])
    out["last_event_id"] = np.array([t.interactions_count for t in trackers])
    out["last_shell_id"] = np.array([t.shell_id for t in trackers])
    out["last_line_absorb_id"] = np.array([t.interaction_line_absorb_id for t in trackers])
    out["last_line_emit_id"] = np.array([t.interaction_line_emit_id for t in trackers])
    for k in ("radius", "before_nu", "before_mu", "before_energy", "after_nu", "after_mu", "after_energy"):
        out["last_" + k] = np.array([getattr(t, k) for t in trackers])
    return out


def run_reference_radfield_nonhomologous(j, nu_bar, j_blue, velocity_gradient, time_of_simulation, volume, line_list_nu,
                                         w_epsilon=1e-10):
    """The unmodified nonhomologous `MCRadiationFieldPropertiesSolver.solve` (modes/nonhomologous/mc_rad_field_solver.py:
    35-131), with the stand-ins of oracle.reference_runner.run_reference_radfield (run once first to install them)."""
    from .reference_loader import _Q
    from .reference_runner import run_reference_radfield

    S, L = len(j), len(line_list_nu)
    run_reference_radfield(np.ones(S), np.ones(S), np.zeros((L, S)), 1.0, 1.0, np.ones(S), line_list_nu)  # installs the stand-ins
    from tardis.transport.montecarlo.estimators.estimators_bulk import EstimatorsBulk
    from tardis.transport.montecarlo.estimators.estimators_line import EstimatorsLine
    from tardis.transport.montecarlo.modes.nonhomologous.mc_rad_field_solver import MCRadiationFieldPropertiesSolver

    bulk = EstimatorsBulk(np.array(j, dtype=np.float64), np.array(nu_bar, dtype=np.float64))
    line = EstimatorsLine(np.array(j_blue, dtype=np.float64), np.zeros_like(j_blue, dtype=np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        out = MCRadiationFieldPropertiesSolver(w_epsilon).solve(bulk, line, np.asarray(velocity_gradient, dtype=np.float64),
                                                               _Q(float(time_of_simulation)), np.asarray(volume, dtype=np.float64),
                                                               np.asarray(line_list_nu, dtype=np.float64))
    st = out.dilute_blackbody_radiationfield_state
    t = st.temperature
    return dict(t_radiative=np.asarray(t.value if isinstance(t, _Q) else t, dtype=np.float64),
                dilution_factor=np.asarray(st.dilution_factor, dtype=np.float64), j_blues=np.asarray(out.j_blues, dtype=np.float64))
