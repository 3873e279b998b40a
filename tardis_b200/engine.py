"""Thin Python owner of one `tb200_engine` (one GPU).  All compute happens in
libtardis_b200.so; this module only marshals NumPy buffers across the C-ABI and
maps error codes to the exception classes the reference raises."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi

LINE_INTERACTION = {"scatter": 0, "downbranch": 1, "macroatom": 2}
SIGMA_THOMSON = 6.652458734e-25  # tardis/transport/montecarlo/configuration/constants.py:3 (CODATA-2010)

EVENT_DTYPE = np.dtype([
    ("packet_id", "i8"), ("interaction_type", "i8"), ("status", "i8"), ("before_shell_id", "i8"),
    ("after_shell_id", "i8"), ("line_absorb_id", "i8"), ("line_emit_id", "i8"),
    ("radius", "f8"), ("before_nu", "f8"), ("before_mu", "f8"), ("before_energy", "f8"),
    ("after_nu", "f8"), ("after_mu", "f8"), ("after_energy", "f8"),
])


class MonteCarloException(ValueError):
    """Same name and base as tardis/transport/montecarlo/utils.py:10."""


class MacroAtomError(ValueError):
    """Same name and base as tardis/transport/montecarlo/macro_atom.py:15."""


class PlasmaException(Exception):
    """Same name and base as tardis/plasma/exceptions.py:1."""


class PlasmaIonizationError(PlasmaException):
    """Same name and base as tardis/plasma/exceptions.py:25 (n_e turned NaN, or did not converge within the device's cap)."""


class EngineError(RuntimeError):
    pass


IONIZATION = {"nebular": 0, "lte": 1}
EXCITATION = {"dilute-lte": 0, "lte": 1}
RADIATIVE_RATES_TYPE = {"dilute-blackbody": 0, "blackbody": 1, "detailed": 2}


_pd = C.POINTER(C.c_double)
_pi = C.POINTER(C.c_int64)


def _dptr(a):
    return a.ctypes.data_as(_pd)


def _iptr(a):
    return a.ctypes.data_as(_pi)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


class Engine:
    """One GPU.  `set_model` once per MC iteration, then `run` (host in / host out) or
    `upload_packets` / `transport` / `sync` / `download` for device-resident work."""

    def __init__(self, device: int = 0):
        self._lib = capi.load()
        self._h = C.c_void_p()
        self._check(self._lib.tb200_create(device, C.byref(self._h)))
        self.device = device
        self._model_shape = None
        self._n_packets = 0
        self._n_continua = 0
        self._n_markov = 0
        self._plasma_shape = None
        self._keep = []

    # ---- plumbing ----
    def _api(self, name: str):
        """The C function `tb200_<name>` that acts on this object's handle (an engine group maps it to `tb200_group_<name>`)."""
        return getattr(self._lib, "tb200_" + name)

    def _check(self, code: int):
        if code == 0:
            return
        msg = (self._lib.tb200_last_error() or b"").decode()
        if code == 1:
            raise MonteCarloException(msg)
        if code == 2:
            raise MacroAtomError(msg)
        if code == 5:
            raise MonteCarloException(msg)
        if code == 6:
            raise PlasmaIonizationError(msg)
        raise EngineError(f"tb200 error {code}: {msg}")

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.tb200_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, name: str, value: int):
        """Tuning knobs of `tb200_set_option`; none of them changes a result.  algorithm (1 jump, 0 scan), pooled (1),
        ctas_per_sm / park_min (0 = measured best for the kernel that will run; each kernel is compiled for its default CTAs
        per SM, so another ctas_per_sm only sizes the grid, at most to what fits), threads_per_cta (256 | 128), vol_min (24),
        refill_min (0 = 12 pooled classic / 8 otherwise), sort_packets (1), sort_bits (5), pipeline_chunks (8), pipeline_edges (1: the first and last
        packet range of `run` are a quarter of the others), keep_opacity_tables (0).  An engine group also takes peer_access
        (1; 0 stages every other member's slice of the collective through cudaMemcpyPeerAsync).  An unknown name raises."""
        self._check(self._api("set_option")(self._h, name.encode(), int(value)))

    # ---- tables ----
    def set_model(self, *, r_inner, r_outer, time_explosion, electron_density, line_list_nu, tau_sobolev,
                  line_interaction_type="scatter", transition_probabilities=None, line2macro_level_upper=None,
                  macro_block_edge_index=None, transition_type=None, destination_level_id=None,
                  transition_line_id=None, spectrum_frequency_grid=None, enable_full_relativity=False,
                  disable_line_scattering=False, sigma_thomson=SIGMA_THOMSON, number_of_vpackets=0,
                  survival_probability=0.0, vpacket_tau_russian=10.0, vpacket_spawn_start_frequency=0.0,
                  vpacket_spawn_end_frequency=1e200, continuum=None, t_electrons=None, luminosity_nu_start=0.0,
                  luminosity_nu_end=np.inf, nonhomologous=False, v_inner=None, v_outer=None):
        """`continuum`: object with the IIP fields of OpacityStateNumbaIIP (bf_threshold_list_nu,
        photo_ion_nu_threshold_mins/maxs, photo_ion_block_references, chi_bf, x_sect, phot_nus, ff_opacity_factor,
        emissivities, photo_ion_activation_idx, k_packet_idx, absorbing_markov_probabilities) -> IIP mode.
        absorbing_markov_probabilities = None (or transition_probabilities = None) leaves the continuum macro atom pending
        until `build_absorbing_markov`.
        `nonhomologous`: the reference's nonhomologous mode, with the piecewise-linear velocity law of the shell-edge
        velocities `v_inner` / `v_outer` [cm / s]; time_explosion is not used there."""
        if nonhomologous and enable_full_relativity:
            raise NotImplementedError("Full relativity not supported for non-homology.")
        if nonhomologous and continuum is not None:
            raise ValueError("continuum processes are not supported in the nonhomologous mode")
        if nonhomologous and (v_inner is None or v_outer is None):
            raise ValueError("the nonhomologous mode needs v_inner and v_outer")
        keep = []
        m = capi.Model()
        r_inner, r_outer, n_e, nu = _f64(r_inner), _f64(r_outer), _f64(electron_density), _f64(line_list_nu)
        # tau_sobolev=None: the opacity tables are built on the device (set_atomic_data + build_opacity)
        tau = None if tau_sobolev is None else np.asarray(tau_sobolev, dtype=np.float64)  # may be a strided view; passed as it lies
        if tau is not None:
            if tau.ndim != 2 or tau.shape != (len(nu), len(r_inner)):
                raise ValueError(f"tau_sobolev must be [n_lines, n_shells], got {tau.shape}")
            if any(s < 0 or s % 8 for s in tau.strides):
                tau = np.ascontiguousarray(tau)
        keep += [r_inner, r_outer, n_e, nu, tau]
        m.n_shells, m.n_lines = len(r_inner), len(nu)
        m.r_inner, m.r_outer, m.electron_density, m.line_list_nu = _dptr(r_inner), _dptr(r_outer), _dptr(n_e), _dptr(nu)
        m.time_explosion = float(time_explosion)
        if tau is not None:
            m.tau_sobolev = _dptr(tau)
            m.tau_line_stride, m.tau_shell_stride = tau.strides[0] // 8, tau.strides[1] // 8
        mode = LINE_INTERACTION[line_interaction_type] if isinstance(line_interaction_type, str) else int(line_interaction_type)
        if mode != 0 or continuum is not None:  # continuum events use the macro atom even when lines scatter coherently
            l2m, edge = _i64(line2macro_level_upper), _i64(macro_block_edge_index)
            tt, dst, tl = _i64(transition_type), _i64(destination_level_id), _i64(transition_line_id)
            keep += [l2m, edge, tt, dst, tl]
            m.n_transitions, m.n_blocks = len(tt), len(edge) - 1
            if transition_probabilities is not None:  # None: built on the device by build_opacity
                tp = np.asarray(transition_probabilities, dtype=np.float64)
                if tp.ndim != 2 or tp.shape != (len(tt), len(r_inner)):
                    raise ValueError("transition_probabilities must be [n_transitions, n_shells]")
                if any(s < 0 or s % 8 for s in tp.strides):
                    tp = np.ascontiguousarray(tp)
                keep.append(tp)
                m.transition_probabilities = _dptr(tp)
                m.tp_transition_stride, m.tp_shell_stride = tp.strides[0] // 8, tp.strides[1] // 8
            m.line2macro_level_upper, m.macro_block_edge_index = _iptr(l2m), _iptr(edge)
            m.transition_type, m.destination_level_id, m.transition_line_id = _iptr(tt), _iptr(dst), _iptr(tl)
        if continuum is not None:
            if t_electrons is None:
                raise ValueError("continuum mode needs t_electrons")
            te = _f64(t_electrons)
            cf = {k: _f64(getattr(continuum, k)) for k in (
                "bf_threshold_list_nu", "photo_ion_nu_threshold_mins", "photo_ion_nu_threshold_maxs", "chi_bf", "x_sect",
                "phot_nus", "ff_opacity_factor", "emissivities", "absorbing_markov_probabilities")
                if k != "absorbing_markov_probabilities" or getattr(continuum, k) is not None}
            ci = {k: _i64(getattr(continuum, k)) for k in ("photo_ion_block_references", "photo_ion_activation_idx")}
            keep += [te] + list(cf.values()) + list(ci.values())
            m.t_electrons = _dptr(te)
            m.n_continua, m.n_phot = len(cf["bf_threshold_list_nu"]), len(cf["phot_nus"])
            for k, v in cf.items():
                setattr(m, k, _dptr(v))
            for k, v in ci.items():
                setattr(m, k, _iptr(v))
            m.n_activation = len(ci["photo_ion_activation_idx"])
            m.k_packet_idx = int(continuum.k_packet_idx)
            if "absorbing_markov_probabilities" in cf:  # otherwise built on the device by build_absorbing_markov
                if cf["absorbing_markov_probabilities"].ndim != 3:
                    raise ValueError("absorbing_markov_probabilities must be [n_shells, n, n]")
                m.n_markov = cf["absorbing_markov_probabilities"].shape[1]
        if v_inner is not None and v_outer is not None:
            vi, vo = _f64(v_inner), _f64(v_outer)
            if len(vi) != len(r_inner) or len(vo) != len(r_inner):
                raise ValueError("v_inner / v_outer must have one entry per shell")
            keep += [vi, vo]
            m.v_inner, m.v_outer = _dptr(vi), _dptr(vo)
        c = capi.Config()
        c.nonhomologous = int(bool(nonhomologous))
        c.continuum_processes_enabled = int(continuum is not None)
        c.enable_full_relativity = int(bool(enable_full_relativity))
        c.line_interaction_type = mode
        c.disable_line_scattering = int(bool(disable_line_scattering))
        c.sigma_thomson = float(sigma_thomson)
        c.number_of_vpackets = int(number_of_vpackets)
        c.survival_probability = float(survival_probability)
        c.vpacket_tau_russian = float(vpacket_tau_russian)
        c.vpacket_spawn_start_frequency = float(vpacket_spawn_start_frequency)
        c.vpacket_spawn_end_frequency = float(vpacket_spawn_end_frequency)
        c.luminosity_nu_start, c.luminosity_nu_end = float(luminosity_nu_start), float(luminosity_nu_end)
        if spectrum_frequency_grid is not None:
            grid = _f64(spectrum_frequency_grid)
            keep.append(grid)
            c.spectrum_frequency_grid = _dptr(grid)
            c.n_grid = len(grid)
        self._check(self._api("set_model")(self._h, C.byref(m), C.byref(c)))
        self._model_shape = (m.n_lines, m.n_shells, int(c.n_grid))
        self._n_transitions = int(m.n_transitions)
        self._n_continua = int(m.n_continua) if continuum is not None else 0

    def set_model_from(self, model, **config):
        """Convenience for `tardis_b200.synthetic.Model`."""
        mac = model.macro
        self.set_model(
            r_inner=model.r_inner, r_outer=model.r_outer, time_explosion=model.time_explosion,
            electron_density=model.electron_density, line_list_nu=model.line_list_nu, tau_sobolev=model.tau_sobolev,
            line_interaction_type=model.line_interaction_type, transition_probabilities=mac.transition_probabilities,
            line2macro_level_upper=mac.line2macro_level_upper, macro_block_edge_index=mac.macro_block_edge_index,
            transition_type=mac.transition_type, destination_level_id=mac.destination_level_id,
            transition_line_id=mac.transition_line_id, spectrum_frequency_grid=model.spectrum_frequency_grid,
            continuum=getattr(model, "continuum", None), t_electrons=model.t_electrons, v_inner=model.v_inner,
            v_outer=model.v_outer, **config)

    # ---- packets ----
    def _packets_struct(self, initial_radii, initial_nus, initial_mus, initial_energies, packet_seeds):
        arrs = [_f64(initial_radii), _f64(initial_nus), _f64(initial_mus), _f64(initial_energies), _i64(packet_seeds)]
        n = len(arrs[1])
        if any(len(a) != n for a in arrs):
            raise ValueError("packet arrays must have equal length")
        pk = capi.Packets()
        pk.n_packets = n
        pk.initial_radii, pk.initial_nus, pk.initial_mus, pk.initial_energies = (_dptr(a) for a in arrs[:4])
        pk.packet_seeds = _iptr(arrs[4])
        return pk, arrs

    def output_shapes(self, n):
        """Shapes of the arrays `run` fills; use to preallocate (e.g. pinned) buffers for `buffers=`."""
        L, S, G = self._model_shape
        return {"output_nus": (n,), "output_energies": (n,), "j": (S,), "nu_bar": (S,), "j_blue": (L, S),
                "edotlu": (L, S), "vhist": (max(G, 1),), "spectrum_emitted": (max(G - 1, 0),),
                "spectrum_reabsorbed": (max(G - 1, 0),), "luminosity_sums": (4,)}

    def _outputs_struct(self, n, *, estimators=True, per_packet=True, track_last_interaction=False, n_tracked_packets=0,
                        max_events_per_packet=0, vlog_capacity=0, buffers=None):
        if self._model_shape is None:
            raise EngineError("set_model first")
        L, S, G = self._model_shape
        res = {}
        o = capi.Outputs()
        shapes = self.output_shapes(n)

        def buf(name):
            if buffers is not None and name in buffers:
                a = buffers[name]
                if a.dtype != np.float64 or a.shape != shapes[name] or not a.flags["C_CONTIGUOUS"]:
                    raise ValueError(f"buffer {name} must be C-contiguous float64 of shape {shapes[name]}")
                return a
            return np.empty(shapes[name])

        if per_packet:  # output_nus / output_energies; False -> only estimators and the fused spectrum come back
            res["output_nus"] = buf("output_nus")
            res["output_energies"] = buf("output_energies")
            o.output_nus, o.output_energies = _dptr(res["output_nus"]), _dptr(res["output_energies"])
        if estimators:
            for k in ("j", "nu_bar", "j_blue", "edotlu", "vhist", "spectrum_emitted", "spectrum_reabsorbed", "luminosity_sums"):
                res[k] = buf(k)
            o.luminosity_sums = _dptr(res["luminosity_sums"])
            o.j, o.nu_bar, o.j_blue, o.edotlu, o.vhist = (_dptr(res[k]) for k in ("j", "nu_bar", "j_blue", "edotlu", "vhist"))
            if G > 1:
                o.spectrum_emitted, o.spectrum_reabsorbed = _dptr(res["spectrum_emitted"]), _dptr(res["spectrum_reabsorbed"])
        if estimators and getattr(self, "_n_continua", 0) > 0:
            nc = self._n_continua
            for k in ("photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator"):
                res[k] = np.zeros((nc, S))
                setattr(o, k, _dptr(res[k]))
            res["ff_heating_estimator"] = np.zeros(S)
            o.ff_heating_estimator = _dptr(res["ff_heating_estimator"])
            res["photo_ion_estimator_statistics"] = np.zeros((nc, S), dtype=np.int64)
            o.photo_ion_estimator_statistics = _iptr(res["photo_ion_estimator_statistics"])
        if track_last_interaction:
            for k in ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id"):
                res[k] = np.empty(n, dtype=np.int64)
                setattr(o, k, _iptr(res[k]))
            for k in ("last_radius", "last_before_nu", "last_before_mu", "last_before_energy", "last_after_nu",
                      "last_after_mu", "last_after_energy"):
                res[k] = np.empty(n)
                setattr(o, k, _dptr(res[k]))
        n_tracked_packets = min(int(n_tracked_packets), n)
        if n_tracked_packets > 0 and max_events_per_packet > 0:
            res["_events"] = np.zeros(n_tracked_packets * max_events_per_packet, dtype=EVENT_DTYPE)
            res["event_counts"] = np.zeros(n_tracked_packets, dtype=np.int64)
            o.events = res["_events"].ctypes.data
            o.event_counts = _iptr(res["event_counts"])
            o.n_tracked_packets, o.max_events_per_packet = n_tracked_packets, max_events_per_packet
        if vlog_capacity > 0:
            for k in ("vlog_nus", "vlog_energies", "vlog_initial_mus", "vlog_initial_rs"):
                res[k] = np.zeros(vlog_capacity)
                setattr(o, k, _dptr(res[k]))
            res["vlog_packet_index"] = np.zeros(vlog_capacity, dtype=np.int64)
            o.vlog_packet_index = _iptr(res["vlog_packet_index"])
            o.vlog_capacity = vlog_capacity
        return o, res

    def _finish(self, o, res):
        res["counters"] = {k: int(getattr(o.counters, k)) for k in capi.COUNTER_FIELDS}
        if "_events" in res:
            nt, cap = o.n_tracked_packets, o.max_events_per_packet
            ev = res.pop("_events").reshape(nt, cap)
            res["events"] = [ev[i, : min(int(res["event_counts"][i]), cap)] for i in range(nt)]
        if o.vlog_capacity > 0:
            res["vlog_count"] = int(o.vlog_count)
        if "vhist" in res and self._model_shape[2] == 0:
            res["vhist"] = res["vhist"][:0]
        return res

    def run(self, initial_radii, initial_nus, initial_mus, initial_energies, packet_seeds, **out_opts):
        """The reference-facing call: host packet arrays in, host results out (`tb200_run`)."""
        pk, keep = self._packets_struct(initial_radii, initial_nus, initial_mus, initial_energies, packet_seeds)
        o, res = self._outputs_struct(pk.n_packets, **out_opts)
        self._check(self._api("run")(self._h, C.byref(pk), C.byref(o)))
        self._n_packets = pk.n_packets
        return self._finish(o, res)

    def run_resident(self, **out_opts):
        """`tb200_run_resident`: the packets already in HBM (`upload_packets` / `create_packets`) through the same pipeline as
        `run` -- per-packet outputs stream back range by range while the next range computes."""
        o, res = self._outputs_struct(self._n_packets, **out_opts)
        self._check(self._api("run_resident")(self._h, C.byref(o)))
        return self._finish(o, res)

    def run_packets(self, packets, **out_opts):
        return self.run(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                        packets.packet_seeds, **out_opts)

    def upload_packets(self, initial_radii, initial_nus, initial_mus, initial_energies, packet_seeds):
        pk, keep = self._packets_struct(initial_radii, initial_nus, initial_mus, initial_energies, packet_seeds)
        self._check(self._api("upload_packets")(self._h, C.byref(pk)))
        self._check(self._api("sync")(self._h))  # host arrays may be released after this
        self._n_packets = pk.n_packets

    def create_packets(self, n_packets: int, seed: int, radius: float, temperature: float, l_samples: int = 1000,
                       max_seed_val: int = 0, beta: float | None = None, weighted: bool = False):
        """Device-side `BlackBodySimpleSource.create_packets` (packet_source/base.py:195-253, black_body.py:122-220) for
        `np.random.default_rng(seed)`, seed = base_seed + seed_offset: the packets are generated in HBM and stay there.
        `weighted=True`: `BlackBodyWeightedSource` (black_body_weighted.py:9-108) -- nus uniform between the extremes of a
        plain black-body draw, energies I(nu) / sum I; needs n_packets >= 1 and no `beta`."""
        l_array = np.cumsum(np.arange(1, l_samples, dtype=np.float64) ** -4)  # black_body.py:166, numpy's own pow
        src = capi.PacketSource()
        src.n_packets = int(n_packets); src.seed = int(seed); src.radius = float(radius); src.temperature = float(temperature)
        src.l_array = l_array.ctypes.data_as(capi._pd); src.n_l = len(l_array); src.max_seed_val = int(max_seed_val)
        if beta is not None:  # BlackBodySimpleSourceRelativistic (black_body_relativistic.py:92-177)
            src.relativistic, src.beta = 1, float(beta)
        src.weighted = int(bool(weighted))
        self._check(self._api("create_packets")(self._h, C.byref(src)))
        self._check(self._api("sync")(self._h))  # l_array may be released after this
        self._n_packets = int(n_packets)

    def download_packets(self):
        """The resident input arrays as a dict (initial_radii, initial_nus, initial_mus, initial_energies, packet_seeds)."""
        n = self._n_packets
        out = {k: np.empty(n, dtype=np.float64) for k in ("initial_radii", "initial_nus", "initial_mus", "initial_energies")}
        out["packet_seeds"] = np.empty(n, dtype=np.int64)
        self._check(self._lib.tb200_download_packets(
            self._h, *(out[k].ctypes.data_as(capi._pd) for k in ("initial_radii", "initial_nus", "initial_mus", "initial_energies")),
            out["packet_seeds"].ctypes.data_as(capi._pi)))
        return out

    def transport(self, zero_estimators: bool = True):
        self._check(self._lib.tb200_transport(self._h, int(zero_estimators)))

    def sync(self):
        self._check(self._lib.tb200_sync(self._h))

    def download(self, **out_opts):
        o, res = self._outputs_struct(self._n_packets, **out_opts)
        self._check(self._lib.tb200_download(self._h, C.byref(o)))
        return self._finish(o, res)

    # ---- opacity build on the device (SURVEY.md §8f rank 3) ----
    def set_atomic_data(self, *, lines_lower_level_index, lines_upper_level_index, g, metastability, wavelength_cm, f_lu, f_ul,
                        energy_lower, energy_upper, nlte_line=None, continuum_rows=None):
        """`tb200_set_atomic_data`: the static per-line / per-level data of the opacity build (once per simulation, after
        the first `set_model`).  `continuum_rows` (continuum mode only, required there): the macro atom's row map, a dict of
        rate_key [T], energy [T], n_rate_rows (6 heights) and n_cooling_rows (3 heights) -- see tb200_continuum_rows;
        `tardis_b200.macro_atom.continuum_row_map` derives it from the reference's metadata."""
        a = capi.AtomicData()
        lo, up = _i64(lines_lower_level_index), _i64(lines_upper_level_index)
        gg = _f64(g)
        meta = np.ascontiguousarray(metastability, dtype=np.uint8)
        wfl = _f64(np.asarray(wavelength_cm, dtype=np.float64) * np.asarray(f_lu, dtype=np.float64))  # (lines.wavelength_cm * lines.f_lu), tau_sobolev.py:56
        flu, ful, elo, eup = _f64(f_lu), _f64(f_ul), _f64(energy_lower), _f64(energy_upper)
        keep = [lo, up, gg, meta, wfl, flu, ful, elo, eup]
        a.n_lines, a.n_levels = len(lo), len(gg)
        a.lines_lower_level_index, a.lines_upper_level_index = _iptr(lo), _iptr(up)
        a.g, a.metastability = _dptr(gg), meta.ctypes.data_as(capi._pu8)
        if nlte_line is not None:
            nl = np.ascontiguousarray(nlte_line, dtype=np.uint8)
            keep.append(nl)
            a.nlte_line = nl.ctypes.data_as(capi._pu8)
        a.wavelength_f_lu, a.f_lu, a.f_ul, a.energy_lower, a.energy_upper = _dptr(wfl), _dptr(flu), _dptr(ful), _dptr(elo), _dptr(eup)
        e_esu, m_e, c, h = 4.80320425e-10, 9.10938291e-28, 2.99792458e10, 6.62606957e-27  # CODATA-2010 cgs (tardis/constants.py:1)
        a.sobolev_coefficient = float((np.pi * e_esu**2) / (m_e * c))          # tau_sobolev.py:9-18
        a.c_einstein = float(4.0 * (np.pi * e_esu) ** 2 / (c * m_e))           # macroatom_line_transitions.py:9-11
        a.c, a.h = c, h
        if continuum_rows is not None:
            key, en = _i64(continuum_rows["rate_key"]), _f64(continuum_rows["energy"])
            if len(key) != len(en):
                raise ValueError("continuum_rows: rate_key and energy need one entry per row")
            cr = capi.ContinuumRows()
            cr.n_transitions, cr.rate_key, cr.energy = len(key), _iptr(key), _dptr(en)
            cr.n_rate_rows[:] = [int(v) for v in continuum_rows["n_rate_rows"]]
            cr.n_cooling_rows[:] = [int(v) for v in continuum_rows["n_cooling_rows"]]
            keep += [key, en, cr]
            a.continuum_rows = C.pointer(cr)
        self._check(self._api("set_atomic_data")(self._h, C.byref(a)))

    def build_opacity(self, level_number_density, time_explosion, j_blues=None, velocity_gradient=None, continuum=None):
        """`tb200_build_opacity`: tau_Sobolev, beta_Sobolev and the normalised macro-atom probabilities of this iteration, built
        in HBM from the level populations [n_levels, S] (`None` outside the continuum mode: the populations `solve_plasma` left
        resident) and J_blue (`None` = the table `solve_radiation_field` or `solve_plasma` left resident).
        `velocity_gradient` [S] (1/s): the nonhomologous mode's tau (modes/nonhomologous/tau_sobolev.py:21-75), required for a
        nonhomologous model, whose `time_explosion` is then not read.  `continuum` (continuum mode only, required there): the
        macro atom's rates of this iteration, a dict of rate (6 arrays [key, S]), cooling (3 arrays [key, S]: the reference's
        cooling arrays transposed), electron_densities, ff_cool_rate, fb_cool_rate, coll_exc_cool_rate, coll_ion_cool_rate
        ([S] each), and optionally beta_sobolev / stimulated_emission_factor [L, S] for the line rows (then
        `level_number_density` is None and tau stays the model's) -- see tb200_continuum_rates.  The normalised table then
        stays in HBM for `build_absorbing_markov(None, ...)`."""
        p = capi.PlasmaState()
        keep = []
        if level_number_density is not None:  # None: continuum["beta_sobolev"] / ["stimulated_emission_factor"] are given
            lnd = _f64(level_number_density)
            keep.append(lnd)
            p.level_number_density = _dptr(lnd)
        p.time_explosion = float(time_explosion)
        if j_blues is not None:
            jb = _f64(j_blues)
            keep.append(jb)
            p.j_blues = _dptr(jb)
        if velocity_gradient is not None:
            g = _f64(velocity_gradient)
            S = self._model_shape[1]
            if g.shape != (S,):
                raise ValueError(f"velocity_gradient must have one entry per shell ({S})")
            keep.append(g)
            p.velocity_gradient = _dptr(g)
        if continuum is not None:
            S = self._model_shape[1]
            cr = capi.ContinuumRates()
            tabs = [_f64(t) for t in (*continuum["rate"], *continuum["cooling"])]
            if len(tabs) != 9 or any(t.ndim != 2 or t.shape[1] != S for t in tabs):
                raise ValueError(f"continuum: 6 rate and 3 cooling tables [key, {S}] are needed")
            shell = [_f64(continuum[k]) for k in ("electron_densities", "ff_cool_rate", "fb_cool_rate", "coll_exc_cool_rate", "coll_ion_cool_rate")]
            if any(a.shape != (S,) for a in shell):
                raise ValueError(f"continuum: the per-shell arrays need {S} entries")
            for k in range(6):
                cr.rate[k] = _dptr(tabs[k])
            for k in range(3):
                cr.cooling[k] = _dptr(tabs[6 + k])
            cr.electron_densities, cr.ff_cool_rate, cr.fb_cool_rate, cr.coll_exc_cool_rate, cr.coll_ion_cool_rate = map(_dptr, shell)
            keep += [*tabs, *shell, cr]
            for k in ("beta_sobolev", "stimulated_emission_factor"):
                if continuum.get(k) is not None:
                    t = _f64(continuum[k])
                    if t.shape != (self._model_shape[0], S):
                        raise ValueError(f"continuum: {k} must be [n_lines, n_shells]")
                    keep.append(t)
                    setattr(cr, k, _dptr(t))
            p.continuum = C.pointer(cr)
        self._check(self._api("build_opacity")(self._h, C.byref(p)))

    # ---- the classic plasma on the device ----
    def set_plasma_data(self, *, level_energy, level_ion, ion_atomic_number, ion_charge, ionization_energy, number_density,
                        zeta_temperatures=None, zeta=None, chi_0=1.9020591570241798e-11):
        """`tb200_set_plasma_data`, once after `set_atomic_data` (whose g and metastability it uses, same level rows): per level
        its excitation energy and ion row, the ion table (atomic number, charge, ionisation energy into the ion; NaN for
        charge 0), number_density [n_elements, S] in the ion table's element order, the zeta table [n_ions, n_T] on its
        temperature grid (nebular ionisation only) and chi_0.  `tardis_b200.plasma.plasma_data` derives all of it from the
        reference's frames."""
        lev_e, lev_ion = _f64(level_energy), _i64(level_ion)
        z, q, chi = _i64(ion_atomic_number), _i64(ion_charge), _f64(ionization_energy)
        nd = _f64(number_density)
        if len(lev_e) != len(lev_ion) or not len(z) == len(q) == len(chi) or nd.ndim != 2:
            raise ValueError("plasma data: one energy and ion row per level, one atomic number / charge / energy per ion, "
                             "number_density [n_elements, n_shells]")
        d = capi.PlasmaData()
        d.n_levels, d.level_energy, d.level_ion = len(lev_e), _dptr(lev_e), _iptr(lev_ion)
        d.n_ions, d.ion_atomic_number, d.ion_charge, d.ionization_energy = len(z), _iptr(z), _iptr(q), _dptr(chi)
        d.n_shells, d.number_density = nd.shape[1], _dptr(nd)
        keep = [lev_e, lev_ion, z, q, chi, nd]
        if zeta is not None:
            zt, zz = _f64(zeta_temperatures), _f64(zeta)
            if zz.shape != (len(z), len(zt)):
                raise ValueError(f"zeta must be [n_ions, n_temperatures] = [{len(z)}, {len(zt)}], got {zz.shape}")
            d.n_zeta_temperatures, d.zeta_temperatures, d.zeta = len(zt), _dptr(zt), _dptr(zz)
            keep += [zt, zz]
        d.chi_0 = float(chi_0)
        d.k_b, d.h, d.m_e, d.c = 1.3806488e-16, 6.62606957e-27, 9.10938291e-28, 2.99792458e10  # CODATA-2010 cgs (tardis/constants.py:1)
        self._check(self._api("set_plasma_data")(self._h, C.byref(d)))
        self._plasma_shape = (len(lev_e), len(z))

    def solve_plasma(self, t_radiative, dilution_factor, *, ionization="nebular", excitation="dilute-lte",
                     radiative_rates_type="dilute-blackbody", link_t_rad_t_electron=0.9, delta_treatment=None,
                     departure_coefficient=None, ion_zero_threshold=1e-20, electron_densities=None, download=False):
        """`tb200_solve_plasma`: level populations, ion populations, n_e and (dilute-blackbody / blackbody) the J_blue table from
        the damped T_rad and W [S].  The populations stay in HBM for `build_opacity(None, ...)`, n_e becomes the model's
        electron densities, J_blue the table `build_opacity(..., j_blues=None)` reads.  `electron_densities` [S]: fixed n_e
        (no fixed point).  A NaN n_e, or no convergence within 1000 iterations, raises PlasmaIonizationError.
        download=True returns a dict of electron_densities [S], ion_number_density [n_ions, S], level_number_density
        [n_levels, S], j_blues [L, S] and iterations; otherwise only iterations."""
        L, S, _ = self._model_shape
        t, w = _f64(t_radiative), _f64(dilution_factor)
        if t.shape != (S,) or w.shape != (S,):
            raise ValueError(f"t_radiative and dilution_factor need one entry per shell ({S})")
        for name, table, v in (("ionization", IONIZATION, ionization), ("excitation", EXCITATION, excitation),
                               ("radiative_rates_type", RADIATIVE_RATES_TYPE, radiative_rates_type)):
            if v not in table:
                raise ValueError(f"{name} must be one of {sorted(table)}, got {v!r}")
        p = capi.PlasmaParams()
        p.t_radiative, p.dilution_factor = _dptr(t), _dptr(w)
        p.ionization, p.excitation = IONIZATION[ionization], EXCITATION[excitation]
        p.radiative_rates_type = RADIATIVE_RATES_TYPE[radiative_rates_type]
        p.link_t_rad_t_electron = float(link_t_rad_t_electron)
        p.delta_treatment = np.nan if delta_treatment is None else float(delta_treatment)
        p.departure_coefficient = np.nan if departure_coefficient is None else float(departure_coefficient)
        p.ion_zero_threshold = float(ion_zero_threshold)
        keep = [t, w]
        if electron_densities is not None:
            ne = _f64(electron_densities)
            if ne.shape != (S,):
                raise ValueError(f"electron_densities needs one entry per shell ({S})")
            keep.append(ne)
            p.electron_densities = _dptr(ne)
        it = C.c_int32(0)
        out = None
        if download:
            n_levels, n_ions = self._plasma_shape
            out = dict(electron_densities=np.empty(S), ion_number_density=np.empty((n_ions, S)),
                       level_number_density=np.empty((n_levels, S)), j_blues=np.empty((L, S)))
        ptr = (lambda k: _dptr(out[k])) if download else (lambda k: None)
        self._check(self._api("solve_plasma")(self._h, C.byref(p), ptr("electron_densities"), ptr("ion_number_density"),
                                              ptr("level_number_density"), ptr("j_blues"), C.byref(it)))
        if out is None:
            return dict(iterations=int(it.value))
        out["iterations"] = int(it.value)
        return out

    def download_opacity(self, transition_probabilities=False):
        """The device-built tables in the reference's host layout: dict of tau_sobolev, beta_sobolev,
        stimulated_emission_factor [L,S] (+ transition_probabilities [T,S] with option keep_opacity_tables = 1)."""
        L, S, _ = self._model_shape
        out = {k: np.empty((L, S)) for k in ("tau_sobolev", "beta_sobolev", "stimulated_emission_factor")}
        tp = np.empty((self._n_transitions, S)) if transition_probabilities else None
        self._check(self._lib.tb200_download_opacity(self._h, _dptr(out["tau_sobolev"]), _dptr(out["beta_sobolev"]),
                                                     _dptr(out["stimulated_emission_factor"]), _dptr(tp) if tp is not None else None))
        if tp is not None:
            out["transition_probabilities"] = tp
        return out

    # ---- the continuum macro atom on the device ----
    def build_absorbing_markov(self, transition_probabilities, source_level_idx, destination_level_idx, transition_type,
                               n_states=None):
        """`tb200_build_absorbing_markov`: the absorbing-Markov-chain table X [S, n, n] and the normalised deactivation table
        of this iteration, built in HBM from the normalised transition probabilities [T, S] (may be a strided view) and the
        rows' source / destination state and type (create_absorbing_probs + the second normalisation of the reference's
        ContinuumMacroAtomSolver).  n_states defaults to max(source_level_idx) + 1.  transition_probabilities = None: the
        table the last continuum-mode `build_opacity` left in HBM."""
        src, dst, tt = _i64(source_level_idx), _i64(destination_level_idx), _i64(transition_type)
        m = capi.MarkovInput()
        keep = [src, dst, tt]
        if transition_probabilities is not None:
            tp = np.asarray(transition_probabilities, dtype=np.float64)
            if tp.ndim != 2:
                raise ValueError("transition_probabilities must be [n_transitions, n_shells]")
            if any(s < 0 or s % 8 for s in tp.strides):
                tp = np.ascontiguousarray(tp)
            if tp.shape[0] != len(src):
                raise ValueError("source_level_idx, destination_level_idx and transition_type need one entry per row")
            if tp.shape[1] != self._model_shape[1]:
                raise ValueError("transition_probabilities must have one column per shell of the model")
            keep.append(tp)
            m.transition_probabilities = _dptr(tp)
            m.tp_transition_stride, m.tp_shell_stride = tp.strides[0] // 8, tp.strides[1] // 8
        if not (len(src) == len(dst) == len(tt)):
            raise ValueError("source_level_idx, destination_level_idx and transition_type need one entry per row")
        m.n_transitions = len(src)
        m.source_level_idx, m.destination_level_idx, m.transition_type = _iptr(src), _iptr(dst), _iptr(tt)
        m.n_states = int(src.max()) + 1 if n_states is None else int(n_states)
        self._check(self._api("build_absorbing_markov")(self._h, C.byref(m)))
        self._n_markov = int(m.n_states)
        del keep

    def download_absorbing_markov(self, matrix=True, deactivating=True):
        """The device-built tables in the reference's host layout: dict of absorbing_markov_probabilities [S, n, n] and the
        normalised deactivating transition_probabilities [T, S]; needs the option keep_opacity_tables = 1 before the build."""
        _, S, _ = self._model_shape
        n = self._n_markov
        out = {}
        if matrix:
            out["absorbing_markov_probabilities"] = np.empty((S, n, n))
        if deactivating:
            out["transition_probabilities"] = np.empty((self._n_transitions, S))
        self._check(self._lib.tb200_download_absorbing_markov(
            self._h, _dptr(out["absorbing_markov_probabilities"]) if matrix else None,
            _dptr(out["transition_probabilities"]) if deactivating else None))
        return out

    # ---- formal-integral source function (SURVEY.md §8f rank 4) ----
    def solve_source_function(self, *, time_explosion, time_of_simulation, volume, wavelength_cm, lines_lower_level_idx,
                              lines_upper_level_idx, n_levels, estimators=None, c=2.99792458e10, tolerance=0.0, max_iterations=0,
                              want=("att_S_ul", "Jred_lu", "Jblue_lu", "e_dot_u")):
        """`tb200_solve_source_function`: att_S_ul, Jred_lu, Jblue_lu [L,S] and e_dot_u [n_levels,S]
        (SourceFunctionSolver.solve, spectrum/formal_integral/source_function.py:27-358) from tau_sobolev, the kept normalised
        transition probabilities (option keep_opacity_tables = 1) and the line estimators resident in HBM after the last
        transport, or from `estimators = (j_blue_estimator[L,S], e_dot_lu_estimator[L,S])` given on the host."""
        L, S, _ = self._model_shape
        p = capi.SourceFunctionParams()
        vol, wave = _f64(volume), _f64(wavelength_cm)
        lo, up = _i64(lines_lower_level_idx), _i64(lines_upper_level_idx)
        if len(vol) != S or len(wave) != L or len(lo) != L or len(up) != L:
            raise ValueError("volume needs one entry per shell, wavelength_cm / level indices one per line")
        keep = [vol, wave, lo, up]
        p.time_explosion, p.time_of_simulation = float(time_explosion), float(time_of_simulation)
        p.volume, p.wavelength_cm = _dptr(vol), _dptr(wave)
        p.lines_lower_level_idx, p.lines_upper_level_idx = _iptr(lo), _iptr(up)
        p.n_levels, p.c = int(n_levels), float(c)
        p.max_iterations, p.tolerance = int(max_iterations), float(tolerance)
        if estimators is not None:
            jb, ed = (_f64(a) for a in estimators)
            if jb.shape != (L, S) or ed.shape != (L, S):
                raise ValueError(f"estimators must be two [n_lines, n_shells] arrays, got {jb.shape}, {ed.shape}")
            keep += [jb, ed]
            p.j_blue_estimator, p.e_dot_lu_estimator = _dptr(jb), _dptr(ed)
        out = {k: np.empty((L, S)) for k in ("att_S_ul", "Jred_lu", "Jblue_lu") if k in want}
        if "e_dot_u" in want:
            out["e_dot_u"] = np.empty((int(n_levels), S))
        it = C.c_int32(0)
        self._check(self._lib.tb200_solve_source_function(
            self._h, C.byref(p), *(_dptr(out[k]) if k in out else None for k in ("att_S_ul", "Jred_lu", "Jblue_lu", "e_dot_u")), C.byref(it)))
        out["iterations"] = int(it.value)
        return out

    # ---- formal integral (SURVEY.md §8f rank 4) ----
    def formal_integral(self, *, inner_temperature, frequencies, points, interpolate_shells=0, tables=None, electron_densities=None,
                        sigma_thomson=0.0, want_intensities=False):
        """`tb200_formal_integral`: luminosity densities [n_frequencies] (and, on request, intensities_nu_p [n_frequencies, points])
        of interpolate_integrator_quantities + numba_formal_integral (spectrum/formal_integral/formal_integral_solver.py:208-285,
        formal_integral_numba.py:377-567) from tau_sobolev / the line list / the geometry of the resident model and the
        att_S_ul, Jred_lu, Jblue_lu tables the last `solve_source_function` left in HBM -- or `tables = (att_S_ul, Jred_lu,
        Jblue_lu)`, each [L,S], given on the host."""
        L, S, _ = self._model_shape
        p = capi.FormalIntegralParams()
        p.inner_temperature = float(inner_temperature)
        p.n_impact_parameters, p.interpolate_shells = int(points), int(interpolate_shells)
        p.sigma_thomson = float(sigma_thomson)
        keep = []
        if tables is not None:
            att, jred, jblue = (_f64(a) for a in tables)
            if att.shape != (L, S) or jred.shape != (L, S) or jblue.shape != (L, S):
                raise ValueError(f"tables must be three [n_lines, n_shells] arrays, got {att.shape}, {jred.shape}, {jblue.shape}")
            keep += [att, jred, jblue]
            p.att_S_ul, p.Jred_lu, p.Jblue_lu = _dptr(att), _dptr(jred), _dptr(jblue)
        if electron_densities is not None:
            ne = _f64(electron_densities)
            if ne.shape != (S,):
                raise ValueError(f"electron_densities must have one entry per shell ({S})")
            keep.append(ne)
            p.electron_densities = _dptr(ne)
        freq = _f64(frequencies)
        if freq.ndim != 1:
            raise ValueError("frequencies must be one-dimensional")
        lum = np.empty(len(freq))
        inup = np.empty((len(freq), int(points))) if want_intensities else None
        self._check(self._api("formal_integral")(self._h, C.byref(p), _dptr(freq), len(freq), _dptr(lum),
                                                    _dptr(inup) if inup is not None else None))
        a, b = C.c_double(0.0), C.c_double(0.0)
        self._check(self._api("formal_integral_ms")(self._h, C.byref(a), C.byref(b)))
        return dict(luminosity_densities=lum, intensities_nu_p=inup, interpolation_ms=a.value, integral_ms=b.value)

    # ---- estimator -> radiation field (SURVEY.md §8f rank 4) ----
    def solve_radiation_field(self, *, time_explosion, time_of_simulation, volume, w_epsilon=1e-10, detailed_optical_window=False,
                              estimators=None, want_j_blues=True, velocity_gradient=None):
        """`tb200_solve_radiation_field`: T_rad, W per shell and the normalised / zero-filled J_blue table
        (MCRadiationFieldPropertiesSolver.solve, mc_rad_field_solver.py:37-144) from the estimators resident in HBM after
        the last transport, or from `estimators = (j, nu_bar, j_blue[L,S])` given on the host.  `velocity_gradient` [S]: the
        nonhomologous mode's solver (modes/nonhomologous/mc_rad_field_solver.py:35-131), required for a nonhomologous model."""
        from scipy.special import zeta  # noqa: PLC0415  (the reference computes its constant with scipy's zeta, :27-29)

        L, S, _ = self._model_shape
        h, k_b, c, sigma_sb = 6.62606957e-27, 1.3806488e-16, 2.99792458e10, 5.670373e-5  # CODATA-2010 cgs (tardis/constants.py:1)
        p = capi.RadfieldParams()
        p.time_explosion, p.time_of_simulation = float(time_explosion), float(time_of_simulation)
        vol = _f64(volume)
        if vol.shape != (S,):
            raise ValueError(f"volume must have one entry per shell ({S})")
        p.volume = _dptr(vol)
        p.w_epsilon, p.detailed_optical_window = float(w_epsilon), int(bool(detailed_optical_window))
        p.t_radiative_estimator_constant = float((np.pi**4 / (15 * 24 * zeta(5, 1))) * (h / k_b))
        p.sigma_sb, p.c, p.h, p.k_b = sigma_sb, c, h, k_b
        keep = [vol]
        if velocity_gradient is not None:
            g = _f64(velocity_gradient)
            if g.shape != (S,):
                raise ValueError(f"velocity_gradient must have one entry per shell ({S})")
            keep.append(g)
            p.velocity_gradient = _dptr(g)
        if estimators is not None:
            j, nu_bar, j_blue = (_f64(a) for a in estimators)
            if j.shape != (S,) or nu_bar.shape != (S,) or j_blue.shape != (L, S):
                raise ValueError("estimators must be (j[S], nu_bar[S], j_blue[L,S])")
            keep += [j, nu_bar, j_blue]
            p.j, p.nu_bar, p.j_blue = _dptr(j), _dptr(nu_bar), _dptr(j_blue)
        t_rad, w = np.empty(S), np.empty(S)
        j_blues = np.empty((L, S)) if want_j_blues else None
        self._check(self._lib.tb200_solve_radiation_field(self._h, C.byref(p), _dptr(t_rad), _dptr(w),
                                                          _dptr(j_blues) if want_j_blues else None))
        return t_rad, w, j_blues

    # ---- measurement / collectives ----
    def last_kernel_ms(self) -> float:
        ms = C.c_double(0)
        self._check(self._lib.tb200_last_kernel_ms(self._h, C.byref(ms)))
        return ms.value

    def counters(self) -> dict:
        c = capi.Counters()
        self._check(self._lib.tb200_get_counters(self._h, C.byref(c)))
        return {k: int(getattr(c, k)) for k in capi.COUNTER_FIELDS}

    def kernel_launches(self) -> int:
        return int(self._lib.tb200_kernel_launches(self._h))

    def estimator_layout(self) -> dict:
        """`tb200_get_estimator_layout`: offsets (in float64) of every table inside the packed estimator buffer."""
        lay = capi.EstimatorLayout()
        self._check(self._lib.tb200_get_estimator_layout(self._h, C.byref(lay)))
        return {k: int(getattr(lay, k)) for k in capi.LAYOUT_FIELDS}

    def line_accumulators(self):
        """`tb200_line_accumulators`: (device pointer, number of int64 words, J_blue scale, Edotlu scale) of the fixed-point
        difference arrays behind J_blue / Edotlu (jump algorithm).  Summing THEM over ranks and calling
        `finalize_line_estimators` makes both tables independent of the number of GPUs, bit for bit."""
        p = C.c_void_p()
        n = C.c_int64()
        s1, s2 = C.c_double(), C.c_double()
        self._check(self._lib.tb200_line_accumulators(self._h, C.byref(p), C.byref(n), C.byref(s1), C.byref(s2)))
        return p.value, n.value, s1.value, s2.value

    def finalize_line_estimators(self) -> None:
        """`tb200_finalize_line_estimators`: difference arrays -> J_blue / Edotlu of the estimator buffer (again)."""
        self._check(self._lib.tb200_finalize_line_estimators(self._h))

    def estimator_buffer(self):
        """(device pointer, number of float64) of the packed estimator buffer (for the all-reduce).  Valid until the next
        `set_model`, which may reallocate it: fetch it again after every `set_model`."""
        p = C.c_void_p()
        n = C.c_int64()
        self._check(self._lib.tb200_estimator_buffer(self._h, C.byref(p), C.byref(n)))
        return p.value, n.value


class _MemberEngine(Engine):
    """One member of an `EngineGroup`: an ordinary engine the group owns (every `Engine` call works on it; closing it only
    drops this handle)."""

    def __init__(self, group: "EngineGroup", handle: C.c_void_p, device: int):
        self._lib = group._lib
        self._h = handle
        self.device = device
        self._group = group  # keeps the owner alive
        self._model_shape = None
        self._n_packets = 0
        self._n_continua = 0
        self._n_markov = 0
        self._plasma_shape = None
        self._keep = []

    def close(self):
        self._h = C.c_void_p()


class EngineGroup(Engine):
    """One MC iteration on several GPUs from one process (`tb200_group_*`): one engine per entry of `devices` (an id may
    repeat: `[0, 0]` is two engines on device 0).  Same methods and result dicts as `Engine`; `run` / `run_resident` shard
    the packets contiguously over the members (`parallel.shard_bounds`), sum the estimators on the devices and return
    J_blue, Edotlu, the counters and every per-packet output bit-identical to one engine over the same packets (J, nu_bar,
    the spectra and the luminosity sums to rounding).  `members` are the engines themselves."""

    def __init__(self, devices):
        devices = [int(d) for d in devices]
        if not devices:
            raise ValueError("an engine group needs at least one device")
        self._lib = capi.load()
        self._h = C.c_void_p()
        self.members = []
        self._check(self._lib.tb200_group_create((C.c_int * len(devices))(*devices), len(devices), C.byref(self._h)))
        self.device = tuple(devices)
        self._model_shape = None
        self._n_packets = 0
        self._n_continua = 0
        self._n_markov = 0
        self._plasma_shape = None
        self._keep = []
        self.last_exact = None  # whether the last collective summed the fixed-point line accumulators
        for i, d in enumerate(devices):
            h = C.c_void_p()
            self._check(self._lib.tb200_group_member(self._h, i, C.byref(h)))
            self.members.append(_MemberEngine(self, h, d))

    def _api(self, name: str):
        return getattr(self._lib, "tb200_group_" + name)

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            for m in self.members:
                m.close()
            self._lib.tb200_group_destroy(self._h)
            self._h = C.c_void_p()

    def shard_bounds(self, n: int):
        """[(lo, hi)] of every member: the rule of `parallel.shard_bounds`."""
        g = len(self.members)
        return [(n * i // g, n * (i + 1) // g) for i in range(g)]

    def _members_hold(self, n: int):
        for m, (lo, hi) in zip(self.members, self.shard_bounds(n)):
            m._n_packets = hi - lo
        self._n_packets = n

    # ---- tables ----
    def set_model(self, **kw):
        super().set_model(**kw)
        for m in self.members:
            m._model_shape, m._n_transitions, m._n_continua = self._model_shape, self._n_transitions, self._n_continua

    def solve_radiation_field(self, **kw):
        """On every member (each keeps the results resident for `build_opacity`); they are identical: member 0's."""
        return [Engine.solve_radiation_field(m, **kw) for m in self.members][0]

    def solve_source_function(self, **kw):
        """On every member (the group's formal integral needs the tables on each); they are identical: member 0's."""
        return [Engine.solve_source_function(m, **kw) for m in self.members][0]

    def download_opacity(self, transition_probabilities=False):
        return self.members[0].download_opacity(transition_probabilities)

    def set_plasma_data(self, **kw):
        super().set_plasma_data(**kw)
        for m in self.members:
            m._plasma_shape = self._plasma_shape

    def build_absorbing_markov(self, *args, **kw):
        """On every member (`tb200_group_build_absorbing_markov`); the members' tables are bit-identical."""
        super().build_absorbing_markov(*args, **kw)
        for m in self.members:
            m._n_markov = self._n_markov

    def download_absorbing_markov(self, matrix=True, deactivating=True):
        return self.members[0].download_absorbing_markov(matrix, deactivating)

    def estimator_layout(self) -> dict:
        return self.members[0].estimator_layout()

    # ---- packets ----
    def run(self, *args, **out_opts):
        res = super().run(*args, **out_opts)
        self._members_hold(self._n_packets)
        self.last_exact = None
        return res

    def upload_packets(self, *args):
        super().upload_packets(*args)
        self._members_hold(self._n_packets)

    def create_packets(self, n_packets: int, *args, **kw):
        super().create_packets(n_packets, *args, **kw)
        self._members_hold(int(n_packets))

    def download_packets(self):
        parts = [m.download_packets() for m in self.members]
        return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}

    def transport(self, zero_estimators: bool = True):
        """`tb200_transport` on every member (members on one device one after the other); then call `allreduce`."""
        busy = {}
        for m in self.members:
            if m.device in busy:
                busy[m.device].sync()
            m.transport(zero_estimators)
            busy[m.device] = m

    def sync(self):
        self._check(self._lib.tb200_group_sync(self._h))

    def allreduce(self) -> bool:
        """`tb200_group_allreduce`: every member ends up with the summed estimators.  True when the fixed-point line
        accumulators were summed (J_blue / Edotlu exact), False when the whole buffer was summed in f64."""
        exact = C.c_int(0)
        self._check(self._lib.tb200_group_allreduce(self._h, C.byref(exact)))
        self.last_exact = bool(exact.value)
        return self.last_exact

    def allreduce_ms(self) -> float:
        ms = C.c_double(0)
        self._check(self._lib.tb200_group_allreduce_ms(self._h, C.byref(ms)))
        return ms.value

    def download(self, *, estimators=True, per_packet=True, buffers=None):
        """After `transport` + `allreduce`: the estimators (member 0's copy) and the per-packet outputs of every member."""
        res = self.members[0].download(estimators=estimators, per_packet=False, buffers=buffers)
        if per_packet:
            parts = [m.download(estimators=False, per_packet=True) for m in self.members]
            for k in ("output_nus", "output_energies"):
                res[k] = np.concatenate([p[k] for p in parts])
        res["counters"] = self.counters()
        return res

    # ---- measurement ----
    def counters(self) -> dict:
        per = [m.counters() for m in self.members]
        return {k: sum(c[k] for c in per) for k in capi.COUNTER_FIELDS}

    def last_kernel_ms(self) -> float:
        """The slowest member's transport kernel time."""
        ran = [m for m in self.members if m._n_packets > 0]
        if not ran:
            raise EngineError("no member has transported packets")
        return max(m.last_kernel_ms() for m in ran)

    def kernel_launches(self) -> int:
        return sum(m.kernel_launches() for m in self.members)

    def _per_member(self, *_a, **_k):
        raise EngineError("a group has one such buffer per member: use group.members[i]")

    line_accumulators = finalize_line_estimators = estimator_buffer = _per_member
