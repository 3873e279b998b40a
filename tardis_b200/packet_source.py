"""Host mirror of the reference's black-body packet source, generating the packets on the GPU.

Mirrors `BlackBodySimpleSource` (tardis/transport/montecarlo/packet_source/black_body.py:19-239) on top of
`BasePacketSource.create_packets` (packet_source/base.py:195-253): same constructor arguments, same
`create_packets(no_of_packets, seed_offset=0)`, `calculate_radfield_luminosity`, `set_temperature_from_luminosity`,
`MAX_SEED_VAL`, `hdf_properties`.  Radii / temperatures are plain cgs numbers (objects with `.cgs.value` / `.value`, such
as astropy quantities, are accepted).  The random stream is numpy's `default_rng(base_seed + seed_offset)`, reproduced on
the device (tardis_b200/csrc/packet_source.cuh): seeds, mus, radii and energies are bit-identical to the reference's, nus
agree to one ulp of `log`.  `legacy_mode_enabled` (the global `np.random` stream of old TARDIS versions) is not offered.
`BlackBodyWeightedSourceB200` mirrors `BlackBodyWeightedSource` (black_body_weighted.py:9-108) the same way.
"""
from __future__ import annotations

import numpy as np

from .montecarlo import PacketCollection

SIGMA_SB = 5.670373e-5  # CODATA-2010 cgs (tardis/constants.py:1)


def _cgs(x) -> float:
    for attr in ("cgs", "value"):
        if hasattr(x, attr):
            x = getattr(x, attr)
    return float(x)


class BlackBodySimpleSourceB200:
    """`packet_source = BlackBodySimpleSourceB200(radius, temperature, base_seed=..., engine=eng)`; after
    `create_packets` the engine holds the packets (as after `Engine.upload_packets`), so the transport can start without
    any host-to-device copy: 40 B per packet that never cross PCIe."""

    MAX_SEED_VAL = 2**32 - 1  # base.py:44
    hdf_properties = ["radius", "temperature", "base_seed"]
    hdf_name = "black_body_simple_source"

    def __init__(self, radius=None, temperature=None, base_seed=None, legacy_mode_enabled=False, legacy_second_seed=None, *, engine=None):
        if legacy_mode_enabled:
            raise NotImplementedError("legacy_mode_enabled draws from the global np.random stream; not offered on the device")
        self.radius = radius
        self.temperature = temperature
        self.base_seed = base_seed
        self.legacy_mode_enabled = False
        self.engine = engine

    @classmethod
    def from_simulation_state(cls, simulation_state, *args, **kwargs):
        """black_body.py:45-66"""
        return cls(simulation_state.r_inner_boundary, simulation_state.t_inner, *args, **kwargs)

    def calculate_radfield_luminosity(self) -> float:
        """base.py:255-277: 4 pi sigma_sb r^2 T^4 [erg/s]"""
        return 4 * np.pi * SIGMA_SB * _cgs(self.radius) ** 2 * _cgs(self.temperature) ** 4

    def set_temperature_from_luminosity(self, luminosity) -> None:
        """black_body.py:221-239"""
        self.temperature = (_cgs(luminosity) / (4 * np.pi * _cgs(self.radius) ** 2 * SIGMA_SB)) ** 0.25

    def create_packets(self, no_of_packets: int, seed_offset: int = 0, *, download: bool = True):
        """base.py:195-253.  `download=False` leaves the arrays on the device only and returns None."""
        if self.radius is None or self.temperature is None:
            raise ValueError("Black body Radius or Temperature isn't set")  # black_body.py:118-120
        if self.base_seed is None:
            raise ValueError("base_seed must be set before creating packets")  # base.py:224-225
        if self.engine is None:
            raise ValueError("BlackBodySimpleSourceB200 needs the Engine that will transport the packets")
        self.engine.create_packets(int(no_of_packets), int(self.base_seed) + int(seed_offset), _cgs(self.radius), _cgs(self.temperature),
                                   max_seed_val=self.MAX_SEED_VAL)
        if not download:
            return None
        a = self.engine.download_packets()
        return PacketCollection(a["initial_radii"], a["initial_nus"], a["initial_mus"], a["initial_energies"], a["packet_seeds"],
                                self.calculate_radfield_luminosity())


class BlackBodySimpleSourceRelativisticB200(BlackBodySimpleSourceB200):
    """`BlackBodySimpleSourceRelativistic` (packet_source/black_body_relativistic.py:19-177) on the device: the inner boundary
    is not comoving with the ejecta, so mu = -beta + sqrt(beta^2 + 2 beta z + z) and the packet energies carry
    (2 beta + 1) / (1 - beta^2) / gamma.  Used by the continuum (IIP) and full-relativity modes."""

    hdf_name = "black_body_simple_source_relativistic"

    def __init__(self, time_explosion=None, **kwargs):
        self.time_explosion = time_explosion
        super().__init__(**kwargs)

    @classmethod
    def from_simulation_state(cls, simulation_state, *args, **kwargs):
        """black_body_relativistic.py:45-70"""
        return cls(simulation_state.time_explosion, radius=simulation_state.r_inner_boundary, temperature=simulation_state.t_inner, *args, **kwargs)

    def create_packets(self, no_of_packets: int, seed_offset: int = 0, *, download: bool = True):
        if self.radius is None or self.time_explosion is None:
            raise ValueError("Black body Radius or Time of Explosion isn't set")  # black_body_relativistic.py:118-121
        if self.temperature is None:
            raise ValueError("Black body Radius or Temperature isn't set")
        if self.base_seed is None:
            raise ValueError("base_seed must be set before creating packets")
        if self.engine is None:
            raise ValueError("BlackBodySimpleSourceRelativisticB200 needs the Engine that will transport the packets")
        self.beta = (_cgs(self.radius) / _cgs(self.time_explosion)) / 2.99792458e10  # :122
        self.engine.create_packets(int(no_of_packets), int(self.base_seed) + int(seed_offset), _cgs(self.radius), _cgs(self.temperature),
                                   max_seed_val=self.MAX_SEED_VAL, beta=self.beta)
        if not download:
            return None
        a = self.engine.download_packets()
        return PacketCollection(a["initial_radii"], a["initial_nus"], a["initial_mus"], a["initial_energies"], a["packet_seeds"],
                                self.calculate_radfield_luminosity())


class BlackBodyWeightedSourceB200(BlackBodySimpleSourceB200):
    """`BlackBodyWeightedSource` (packet_source/black_body_weighted.py:9-108) on the device: nus uniform between the min
    and max of a plain black-body draw, each packet's energy I(nu) / sum I with I the Planck intensity, so the Wien tail
    and the far red are sampled as densely as the peak.  Constructed by keyword only, as the reference class.  After a
    download `self.nus` holds the frequencies, as the reference leaves them.  Seeds, radii and mus are bit-identical to
    the reference's; nus and energies agree to the bounds INTEGRATION.md states (ulps of log, pow and exp)."""

    hdf_properties = ["radius", "temperature", "base_seed"]
    hdf_name = "black_body_weighted_source"

    def __init__(self, **kwargs):
        super().__init__(**kwargs)

    def create_packets(self, no_of_packets: int, seed_offset: int = 0, *, download: bool = True):
        """base.py:195-253 with black_body_weighted.py:55-108.  `download=False` leaves the arrays on the device only and
        returns None."""
        if self.radius is None or self.temperature is None:
            raise ValueError("Black body Radius or Temperature isn't set")
        if self.base_seed is None:
            raise ValueError("base_seed must be set before creating packets")
        if int(no_of_packets) == 0:  # nus.min() of the reference
            raise ValueError("zero-size array to reduction operation minimum which has no identity")
        if self.engine is None:
            raise ValueError("BlackBodyWeightedSourceB200 needs the Engine that will transport the packets")
        self.__dict__.pop("nus", None)
        self.engine.create_packets(int(no_of_packets), int(self.base_seed) + int(seed_offset), _cgs(self.radius), _cgs(self.temperature),
                                   max_seed_val=self.MAX_SEED_VAL, weighted=True)
        if not download:
            return None
        a = self.engine.download_packets()
        self.nus = a["initial_nus"]
        return PacketCollection(a["initial_radii"], a["initial_nus"], a["initial_mus"], a["initial_energies"], a["packet_seeds"],
                                self.calculate_radfield_luminosity())
