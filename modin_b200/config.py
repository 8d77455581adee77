"""Configuration knobs of the B200 execution, mirroring the subset of ``modin.config`` that the
partition-execution path reads (modin/config/envvars.py):

* ``NPartitions``          envvars.py:837-885  -- row partitions per frame; the reference defaults to
  the CPU count, here the default is ONE partition per GPU (a partition is a whole device shard);
* ``MinRowPartitionSize`` / ``MinColumnPartitionSize`` envvars.py:1149-1190 (both 32);
* ``BenchmarkMode``        envvars.py:950-968   -- block until device work is finished after every
  partition-manager call;
* ``GpuCount``             envvars.py:818-821.

Each is a tiny ``Parameter`` with ``get``/``put`` and an environment default (``MODIN_*``), the
same surface the reference's pub-sub parameters expose (modin/config/pubsub.py).
"""

from __future__ import annotations

import os


class Parameter:
    varname: str = ""
    default = None
    type = int
    _value = None

    @classmethod
    def get(cls):
        if cls._value is None:
            raw = os.environ.get(cls.varname)
            if raw is not None:
                cls._value = cls._parse(raw)
            else:
                cls._value = cls._get_default()
        return cls._value

    @classmethod
    def put(cls, value):
        cls._value = cls._parse(value) if isinstance(value, str) else cls.type(value)

    @classmethod
    def _parse(cls, raw):
        if cls.type is bool:
            return str(raw).strip().lower() in ("1", "true", "yes", "on")
        return cls.type(raw)

    @classmethod
    def _get_default(cls):
        return cls.default


class GpuCount(Parameter):
    """Number of GPUs the job runs on (= torch.distributed world size; 1 without it)."""

    varname = "MODIN_GPUS"

    @classmethod
    def _get_default(cls):
        return int(os.environ.get("WORLD_SIZE", "1"))


class NPartitions(Parameter):
    """Row partitions per frame ON THIS RANK (reference: total partitions = CpuCount)."""

    varname = "MODIN_NPARTITIONS"
    default = 1

    @classmethod
    def put(cls, value):
        value = int(value)
        if value <= 0:
            raise ValueError(f"NPartitions should be > 0, passed value {value}")
        cls._value = value


class MinRowPartitionSize(Parameter):
    varname = "MODIN_MIN_ROW_PARTITION_SIZE"
    default = 32


class MinColumnPartitionSize(Parameter):
    varname = "MODIN_MIN_COLUMN_PARTITION_SIZE"
    default = 32


class BenchmarkMode(Parameter):
    varname = "MODIN_BENCHMARK_MODE"
    default = False
    type = bool


class ReduceVariant(Parameter):
    """0 = TMA-staged shared-memory tiles (default), 1 = direct 128-bit loads."""

    varname = "MB200_REDUCE_VARIANT"
    default = 0


class HostStreamMinBytes(Parameter):
    """Host frames whose blocks are at least this large stay on the HOST at ingest (``HostBlock``): a fusable
    elementwise call queue followed by ``to_pandas`` is then streamed chunk by chunk through the device
    (``mb200_map_host``: H2D / kernel / D2H overlapped), and anything else copies the block to the device first.
    0 disables (every ingest is an immediate H2D copy)."""

    varname = "MB200_HOST_STREAM_MIN_BYTES"
    default = 64 << 20


class GroupbyDenseKeys(Parameter):
    """Use a direct-addressed (dense) group table when the key range is narrow (default on);
    off = always hash.  The choice reads the key column's cached statistics (``KeyStats``: left behind by the kernel
    that produced the column; one 8 B/row pass, once, for a column of unknown origin)."""

    varname = "MB200_GB_DENSE"
    default = True
    type = bool


class GroupbyAsyncEmit(Parameter):
    """Dense group tables are emitted without a host round trip (the result block is sized on the device and reads
    its row count back lazily); off = count first, then emit exactly that many rows."""

    varname = "MB200_GB_ASYNC_EMIT"
    default = True
    type = bool


class GroupbyDistinctBytes(Parameter):
    """Device bytes one column batch of ``groupby.nunique`` may give its distinct set (16 B per slot, at least twice as
    many slots as the batch has values).  Wider frames run in more batches, each with its own pass over the keys; one
    column always runs, even when its set alone is larger."""

    varname = "MB200_GB_DISTINCT_BYTES"
    default = 8 << 30
