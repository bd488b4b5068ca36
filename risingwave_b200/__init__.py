"""risingwave_b200 -- H100-native (sm_90a) streaming HashAgg / HashJoin / hash-shuffle path behind
RisingWave's executor interface.  See DESIGN.md for scope; include/rwgpu.h is the drop-in C ABI."""
from . import abi  # noqa: F401
from .stream_chunk import StreamChunk, Column  # noqa: F401
from .executor import (AggCall, Backend, Barrier, HashAggExecutor, HashJoinExecutor, JoinParams,  # noqa: F401
                       Message, MessageSender, MessageStream, MockSource, Watermark, PENDING)

__version__ = "0.1.0"
