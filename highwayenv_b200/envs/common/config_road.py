"""The part of a network env whose lane table and population follow its config (roundabout-generic, merge-generic).

Such an env builds its road from config keys (a cached ``NetworkTable`` per key), so two envs of one class may run
different tables; its population is ``N_VEHICLES`` slots' worth at most, and the device reset may place fewer (a
vehicle whose tries all fail is skipped), so the state carries a per-env ``count`` on either slot stride.
"""
from __future__ import annotations

import numpy as np
import torch

from ... import _native as N
from ...road.network import NetworkTable


class ConfigRoadMixin:
    """Mixed in before a ``BatchedNetworkEnv`` family class.  ``define_spaces`` of the class calls ``_use_road`` with
    the table of its config and its largest population before the family's own ``define_spaces``; a new table (another
    config, or ``reset(options={"config": ...})``) drops the device copy so that it is rebuilt."""

    ROAD_KEYS: tuple = ()  # the config keys the lane table depends on (named in copy_envs' refusal)

    def _use_road(self, road: NetworkTable, n_vehicles: int) -> None:
        if self._net is not road:
            self._net = None
        self._road = road
        self.N_VEHICLES = n_vehicles
        self.SLOTS = N.HWY_NET_GROUP if n_vehicles <= N.HWY_NET_GROUP else N.HWY_NET_GROUP_LARGE

    def _make_network(self) -> NetworkTable:
        return self._road

    def _allocate(self) -> None:
        super()._allocate()  # the 32-slot state already carries the population and the (unused) rule clock
        if self.vp == N.HWY_NET_GROUP:  # the 8-slot kernels read the population when the state carries one
            self._count = torch.full((self.num_envs,), self.N_VEHICLES, dtype=torch.int32, device=self.device)
            self._state.count = self._count.data_ptr()
            self._road_steps = None

    def to_finite_mdp(self):
        raise NotImplementedError(f"to_finite_mdp on {self.ENV_ID}")

    def copy_envs(self, dst_ids, src_ids, source=None) -> None:
        """BatchedVectorEnv.copy_envs; two envs of one class may still run different lane tables or slot strides,
        and a state only means something on its own table."""
        if source is not None and type(source) is type(self) and (source._road is not self._road
                                                                   or source.vp != self.vp):
            raise ValueError(f"copy_envs between {self.ENV_ID} envs on different roads ({', '.join(self.ROAD_KEYS)}) "
                             "or slot strides")
        super().copy_envs(dst_ids, src_ids, source)

    def state_dict(self) -> dict:
        """The family's fields [N, V]; `count` vehicles of each env are on the road."""
        sd = super().state_dict()
        sd["count"] = self._count.cpu().numpy()
        return sd

    def load_state_dict(self, sd: dict, env_ids=None) -> None:
        super().load_state_dict(sd, env_ids)
        idx = slice(None) if env_ids is None else torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(self.device)
        self._count[idx] = torch.from_numpy(np.asarray(sd["count"], dtype=np.int32).reshape(-1)).to(self.device)
        if self._road_steps is not None:
            self._road_steps[idx] = 0
