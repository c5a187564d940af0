"""torchstore_b200 -- H100-native weight-sync path behind torchstore's API.

``import torchstore_b200 as ts`` gives the reference package's public names (torchstore/__init__.py:47-69):
store lifecycle (initialize, initialize_spmd, shutdown, client, reset_client), key/value calls (put, get, put_batch,
get_batch, delete, delete_batch, keys, exists), state dicts (put_state_dict, get_state_dict), strategies and
init_logging -- plus TransportType / TensorSlice / Request, which callers of the NVLink transport need.
"""

from torchstore_b200 import api as _api, spmd
from torchstore_b200.logging import init_logging
from torchstore_b200.strategy import ControllerStorageVolumes, HostStrategy, LocalRankStrategy, TorchStoreStrategy
from torchstore_b200.transport import TransportType
from torchstore_b200.transport.types import Request, TensorSlice

_API_NAMES = (
    "initialize shutdown client reset_client "
    "put get put_batch get_batch delete delete_batch keys exists "
    "put_state_dict get_state_dict"
).split()
globals().update({name: getattr(_api, name) for name in _API_NAMES})

initialize_spmd = spmd.initialize
api = _api

__all__ = sorted(
    _API_NAMES
    + ["initialize_spmd", "init_logging", "spmd", "TorchStoreStrategy", "LocalRankStrategy", "HostStrategy",
       "ControllerStorageVolumes", "TransportType", "TensorSlice", "Request"]
)
