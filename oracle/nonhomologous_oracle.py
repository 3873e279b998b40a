"""ctypes front-end of the nonhomologous CPU oracle (oracle/nonhomologous_oracle.cpp).

TEST INFRASTRUCTURE ONLY: compiled with g++ -O2 -ffp-contract=off into tests/_shim on first use (the source includes the
product's header tardis_b200/csrc/nonhomologous.cuh, so the quartic is the device's).  Inputs and outputs are those of
oracle.cpu_oracle.run_oracle, plus the model's v_inner / v_outer.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .cpu_oracle import EVENT_DTYPE, LINE_INTERACTION, OracleError, _Config, _Counters, _d, _i, _Model, _Outputs, _Packets, _pd, _pi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "nonhomologous_oracle.cpp")
HDR = os.path.join(ROOT, "tardis_b200", "csrc", "nonhomologous.cuh")
LIB = os.path.join(ROOT, "tests", "_shim", "libnonhomologous_oracle.so")

_lib = None


def lib():
    global _lib
    if _lib is None:
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        deps = [SRC, HDR, os.path.join(HERE, "tardis_oracle.h")]
        if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(d) for d in deps):
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-o", LIB, SRC],
                           check=True)
        _lib = C.CDLL(LIB)
        _lib.nonhomologous_oracle_run.restype = C.c_int
        _lib.nonhomologous_oracle_run.argtypes = [C.POINTER(_Model), _pd, _pd, C.POINTER(_Config), C.POINTER(_Packets),
                                                  C.POINTER(_Outputs)]
        _lib.nonhomologous_oracle_velocity_gradient.restype = C.c_double
        _lib.nonhomologous_oracle_velocity_gradient.argtypes = [C.c_double] * 4
    return _lib


def velocity_gradient(model):
    f = lib().nonhomologous_oracle_velocity_gradient
    return np.array([f(a, b, c, d) for a, b, c, d in zip(model.r_inner, model.r_outer, model.v_inner, model.v_outer)])


def run_oracle(model, packets, *, number_of_vpackets=0, disable_line_scattering=False, survival_probability=0.0,
               vpacket_tau_russian=10.0, spawn_start=0.0, spawn_end=1e200, sigma_thomson=6.652458734e-25,
               n_tracked_packets=0, max_events_per_packet=512, vlog_capacity=0):
    """One MC iteration of the nonhomologous mode on the CPU; keys as oracle.cpu_oracle.run_oracle."""
    L = lib()
    keep = []
    m = _Model()
    m.n_shells, m.n_lines = model.n_shells, model.n_lines
    for name in ("r_inner", "r_outer", "electron_density", "line_list_nu", "tau_sobolev"):
        a, p = _d(getattr(model, name)); keep.append(a); setattr(m, name, p)
    m.time_explosion = 0.0
    mac = model.macro
    a, p = _d(mac.transition_probabilities); keep.append(a); m.transition_probabilities = p
    m.n_transitions, m.n_blocks = mac.transition_probabilities.shape[0], len(mac.macro_block_edge_index) - 1
    for name in ("line2macro_level_upper", "macro_block_edge_index", "transition_type", "destination_level_id", "transition_line_id"):
        a, p = _i(getattr(mac, name)); keep.append(a); setattr(m, name, p)
    vi, pvi = _d(model.v_inner); vo, pvo = _d(model.v_outer); keep += [vi, vo]
    c = _Config()
    c.line_interaction_type = LINE_INTERACTION[model.line_interaction_type]
    c.disable_line_scattering = int(disable_line_scattering)
    c.sigma_thomson = sigma_thomson
    c.number_of_vpackets = number_of_vpackets
    c.survival_probability = survival_probability
    c.vpacket_tau_russian = vpacket_tau_russian
    c.vpacket_spawn_start_frequency, c.vpacket_spawn_end_frequency = spawn_start, spawn_end
    a, p = _d(model.spectrum_frequency_grid); keep.append(a); c.spectrum_frequency_grid = p
    c.n_grid = len(model.spectrum_frequency_grid)
    pk = _Packets()
    n = len(packets)
    pk.n_packets = n
    for name in ("initial_radii", "initial_nus", "initial_mus", "initial_energies"):
        a, p = _d(getattr(packets, name)); keep.append(a); setattr(pk, name, p)
    a, p = _i(packets.packet_seeds); keep.append(a); pk.packet_seeds = p
    S, Ln = model.n_shells, model.n_lines
    res = dict(output_nus=np.empty(n), output_energies=np.empty(n), j=np.zeros(S), nu_bar=np.zeros(S),
               j_blue=np.zeros((Ln, S)), edotlu=np.zeros((Ln, S)), vhist=np.zeros(c.n_grid))
    o = _Outputs()
    for k, v in res.items():
        setattr(o, k, v.ctypes.data_as(_pd))
    for k in ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id"):
        res[k] = np.empty(n, dtype=np.int64); setattr(o, k, res[k].ctypes.data_as(_pi))
    for k in ("last_radius", "last_before_nu", "last_before_mu", "last_before_energy", "last_after_nu", "last_after_mu", "last_after_energy"):
        res[k] = np.empty(n); setattr(o, k, res[k].ctypes.data_as(_pd))
    n_tracked_packets = min(n_tracked_packets, n)
    if n_tracked_packets > 0:
        ev = np.zeros(n_tracked_packets * max_events_per_packet, dtype=EVENT_DTYPE)
        evc = np.zeros(n_tracked_packets, dtype=np.int64)
        o.events, o.event_counts = ev.ctypes.data, evc.ctypes.data_as(_pi)
        o.n_tracked_packets, o.max_events_per_packet = n_tracked_packets, max_events_per_packet
    if vlog_capacity > 0:
        for k in ("vlog_nus", "vlog_energies", "vlog_initial_mus", "vlog_initial_rs"):
            res[k] = np.zeros(vlog_capacity); setattr(o, k, res[k].ctypes.data_as(_pd))
        res["vlog_packet_index"] = np.zeros(vlog_capacity, dtype=np.int64)
        o.vlog_packet_index, o.vlog_capacity = res["vlog_packet_index"].ctypes.data_as(_pi), vlog_capacity
    err = L.nonhomologous_oracle_run(C.byref(m), pvi, pvo, C.byref(c), C.byref(pk), C.byref(o))
    if err:
        raise OracleError({2: "MacroAtomError", 3: "vpacket did not terminate"}.get(err, str(err)))
    res["counters"] = {k: getattr(o.counters, k) for k, _ in _Counters._fields_}
    if n_tracked_packets > 0:
        ev = ev.reshape(n_tracked_packets, max_events_per_packet)
        res["events"] = [ev[i, : evc[i]] for i in range(n_tracked_packets)]
        res["event_counts"] = evc
    if vlog_capacity > 0:
        res["vlog_count"] = o.vlog_count
    return res


def solve_radiation_field(j, nu_bar, j_blue, velocity_gradient, time_of_simulation, volume, line_list_nu, w_epsilon=1e-10):
    """modes/nonhomologous/mc_rad_field_solver.py:35-131 -> (t_radiative[S], dilution_factor[S], j_blues[L,S])"""
    from .radfield_oracle import C, SIGMA_SB, T_RADIATIVE_ESTIMATOR_CONSTANT, intensity_black_body

    j, nu_bar, j_blue, volume, g = (np.asarray(a, dtype=np.float64) for a in (j, nu_bar, j_blue, volume, velocity_gradient))
    t_rad = T_RADIATIVE_ESTIMATOR_CONSTANT * nu_bar / j
    w = j / (4 * SIGMA_SB * t_rad**4 * time_of_simulation * volume)
    with np.errstate(divide="ignore", invalid="ignore"):
        norm = C / g / (4 * np.pi * time_of_simulation * volume)                        # :120-124
        j_blues = j_blue * norm
    planck = w * intensity_black_body(np.asarray(line_list_nu)[np.newaxis].T, t_rad)
    zero = j_blues == 0.0
    j_blues[zero] = w_epsilon * planck[zero]
    return t_rad, w, j_blues
