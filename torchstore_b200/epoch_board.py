"""Epoch board: the controller's index epoch and every volume's layout epoch in ONE page of POSIX
shared memory, so a client on the same box validates a replayable put/get session with two memory
loads instead of two RPC round trips (storage_volume.py ``InMemoryStore.epoch``, controller.py
``Controller.epoch``; see fast_lane.py).

Slot 0 belongs to the controller, slot 1+i to volume i.  Each slot has exactly one writer (the process
that owns the controller / the volume), which stores the new value *inside* the endpoint that changes
the layout, before that endpoint returns -- so a reader can never see an epoch older than what an RPC
issued at the same moment would have reported.  Aligned 8-byte loads and stores are single instructions.

The board is an optimisation: when it cannot be created or attached the epochs are read by RPC.
The segment is created with the host tier's ``tsb_shm_create`` (include/tstore_b200.h).
"""

from __future__ import annotations

import ctypes
import logging
import os

from torchstore_b200 import _native

logger = logging.getLogger(__name__)

BOARD_BYTES = 4096
MAX_SLOTS = BOARD_BYTES // 8


def reap_stale_segments() -> int:
    """Unlink /dev/shm segments of this library whose creating process is gone (a killed job cannot
    unlink its own): names are tsb200_<pid>_... and tsb200_epochs_<pid>_....  Returns how many went."""
    import re

    gone = 0
    try:
        names = os.listdir("/dev/shm")
    except OSError:
        return 0
    for name in names:
        m = re.match(r"tsb200_(?:epochs_)?(\d+)_", name)
        if not m:
            continue
        pid = int(m.group(1))
        try:
            os.kill(pid, 0)
            continue  # creator alive
        except ProcessLookupError:
            pass
        except PermissionError:
            continue  # alive, someone else's
        try:
            os.unlink(os.path.join("/dev/shm", name))
            gone += 1
        except OSError:
            pass
    return gone


class EpochBoard:
    def __init__(self, name: str, ptr: int, owner: bool):
        self.name, self._ptr, self._owner = name, ptr, owner
        self._slots = (ctypes.c_uint64 * MAX_SLOTS).from_address(ptr)

    @classmethod
    def create(cls) -> "EpochBoard | None":
        name = f"/tsb200_epochs_{os.getpid()}_{os.urandom(4).hex()}"
        reap_stale_segments()
        try:
            ptr = _native.shm_create(name, BOARD_BYTES)
        except Exception as e:  # no /dev/shm, library missing ...: epochs travel by RPC
            logger.debug("epoch board not available: %s", e)
            return None
        board = cls(name, ptr, owner=True)
        ctypes.memset(ptr, 0, BOARD_BYTES)
        return board

    @classmethod
    def attach(cls, name: str) -> "EpochBoard | None":
        try:
            return cls(name, _native.shm_attach(name, BOARD_BYTES), owner=False)
        except Exception as e:
            logger.debug("epoch board %s not attachable: %s", name, e)
            return None

    def write(self, slot: int, value: int) -> None:
        if self._slots is not None:
            self._slots[slot] = value

    def read(self, slot: int) -> int:
        """-1 once the board is closed (never equal to a recorded epoch: sessions fall back to the slow path)."""
        return int(self._slots[slot]) if self._slots is not None else -1

    def close(self) -> None:
        if self._ptr:
            self._slots = None
            try:
                _native.shm_detach(self._ptr, BOARD_BYTES)
                if self._owner:
                    _native.shm_unlink(self.name)
            except Exception as e:
                logger.debug("epoch board close: %s", e)
            self._ptr = 0


_attached: dict[str, EpochBoard] = {}


def attached(name: str | None) -> EpochBoard | None:
    """Process-wide cache of attachments (one mapping per board per process, shared by the client
    and the volumes that live in it)."""
    if not name:
        return None
    board = _attached.get(name)
    if board is None:
        board = EpochBoard.attach(name)
        if board is not None:
            _attached[name] = board
    return board


def forget(name: str | None) -> None:
    """Drop this process's attachment (store shutdown).  Holders that still reference the object see
    a closed board: writes are ignored, reads return -1."""
    board = _attached.pop(name, None) if name else None
    if board is not None:
        board.close()
