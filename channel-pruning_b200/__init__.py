"""cpb200 -- H100-native channel-pruning solver (hot path of ethanhe42/channel-pruning).

The directory name carries a hyphen (it mirrors the reference repo's name), so import it as
``import cpb200`` (alias module at the repo root) or ``importlib.import_module
("channel-pruning_b200")``.  Sub-modules:

  _cabi     cffi binding of libcpb200.so (include/cpb200.h)
  engine    torch-tensor plumbing around the C ABI (streams, handles)
  lib       drop-in mirror of the reference's lib.decompose / lib.net / lib.cfgs
  pruner    multi-layer pipeline + multi-GPU layer sharding (one all_gather)
  synth     synthetic VGG-16 layer problems (BASELINE.json configs)
"""
import os as _os

# One stream per layer problem (13+ in flight) needs as many hardware work queues: with the default 8 the
# streams alias and a stream waiting on its transfer stalls unrelated layers.
# Read by the driver when the CUDA context is created, so it must be set before the first CUDA call.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

from . import _cabi, engine, synth, pruner  # noqa: F401,E402
from . import lib  # noqa: F401,E402
from .engine import Engine, get_engine, reset_engine  # noqa: F401,E402

__version__ = "0.1.0"
