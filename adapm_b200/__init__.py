"""adapm_b200 - a GPU-native (Hopper, sm_90a), intent-driven parameter manager.

Python API with the reference's method names (``bindings/bindings.cc:79-374`` of
alexrenz/AdaPM): ``setup``, ``scheduler``, ``Server``, ``Worker`` with
``pull / push / set / intent / advance_clock / current_clock / prepare_sample /
pull_sample / begin_setup / end_setup / wait_sync / barrier / wait / waitall /
finalize / get_key_size / num_keys``.

Differences that follow from the GPU-first design:

* one process per GPU (``torchrun``); there is no scheduler process - ``scheduler()``
  returns immediately and exists only so that reference launch scripts keep working;
* keys/values may be CUDA tensors (the op is enqueued on the current CUDA stream and
  is asynchronous) or CPU tensors / NumPy arrays (staged through pinned memory);
* ``async`` became a Python keyword after the reference was written, the flag is
  called ``asynchronous`` here (third positional argument, as in the reference).
"""
from __future__ import annotations

import os
import threading
from typing import Optional, Sequence, Union

import numpy as np
import torch

try:
    from . import _C
except ImportError:  # pragma: no cover - first use in a fresh checkout
    from . import _build as _b

    _b.build()
    from . import _C

LOCAL = _C.LOCAL
CLOCK_MAX = _C.CLOCK_MAX
AdapmError = _C.AdapmError

_DTYPES = {"float32": torch.float32, "float64": torch.float64, "int64": torch.int64}

_setup_lock = threading.Lock()
_setup = {"num_keys": None, "num_threads": 1, "techniques": "", "num_channels": -1, "options": {}}


def _env_int(*names: str, default: Optional[int] = None) -> Optional[int]:
    for n in names:
        v = os.environ.get(n)
        if v is not None and v != "":
            return int(v)
    return default


def default_job() -> str:
    j = os.environ.get("ADAPM_JOB")
    if j:
        return j
    port = os.environ.get("MASTER_PORT") or os.environ.get("DMLC_PS_ROOT_PORT") or "0"
    return f"{port}_{os.getppid()}"


def setup(num_keys: int, num_threads: int, use_techniques: str = "", num_channels: int = -1, **options) -> None:
    """Configure the parameter manager (reference ``adapm.setup``, bindings.cc:18-31).

    ``options`` takes every reference flag by name, e.g. ``**{"sys.sync.max_per_sec": 200}``.
    """
    with _setup_lock:
        _setup["num_keys"] = int(num_keys)
        _setup["num_threads"] = int(num_threads)
        _setup["techniques"] = use_techniques
        _setup["num_channels"] = int(num_channels)
        _setup["options"] = {str(k): str(v) for k, v in options.items()}


def scheduler(num_keys: int = 0, num_threads: int = 0) -> None:
    """No-op: membership and barriers run through the shared control block (control.h)."""
    return None


def _as_keys(keys) -> torch.Tensor:
    if isinstance(keys, np.ndarray):
        keys = torch.from_numpy(np.ascontiguousarray(keys))
    elif not isinstance(keys, torch.Tensor):
        keys = torch.as_tensor(keys, dtype=torch.int64)
    if keys.dtype != torch.int64:
        keys = keys.to(torch.int64)
    return keys.contiguous().view(-1)


class Server:
    """One parameter-server node = one rank = one GPU (reference ``adapm.Server``)."""

    def __init__(
        self,
        value_lengths: Union[int, torch.Tensor, np.ndarray, Sequence[int]],
        *,
        num_keys: Optional[int] = None,
        num_threads: Optional[int] = None,
        rank: Optional[int] = None,
        world: Optional[int] = None,
        backend: Optional[str] = None,
        fabric: Optional[str] = None,
        job: Optional[str] = None,
        dtype: str = "float32",
        device: Optional[int] = None,
        options: Optional[dict] = None,
    ) -> None:
        with _setup_lock:
            cfg = dict(_setup)
        world = world if world is not None else _env_int("WORLD_SIZE", "OMPI_COMM_WORLD_SIZE", "PMI_SIZE", "SLURM_NTASKS",
                                                         "DMLC_NUM_SERVER", default=1)
        rank = rank if rank is not None else _env_int("RANK", "OMPI_COMM_WORLD_RANK", "PMI_RANK", "SLURM_PROCID",
                                                      "DMLC_RANK", default=0)
        if backend is None:
            backend = os.environ.get("ADAPM_BACKEND") or ("cuda" if (_C.cuda_available() and dtype == "float32") else "cpu")
        if fabric is None:
            fabric = os.environ.get("ADAPM_FABRIC") or ("shm" if world > 1 else "inproc")
        opts = {"backend": backend, "fabric": fabric, "rank": rank, "world": world, "dtype": dtype,
                "job": job or default_job(), "workers": num_threads if num_threads is not None else cfg["num_threads"]}
        if device is not None:
            opts["device"] = device
        elif backend == "cuda":
            lr = _env_int("LOCAL_RANK", "OMPI_COMM_WORLD_LOCAL_RANK", "SLURM_LOCALID")
            if lr is not None and fabric == "shm":
                opts["device"] = lr % max(1, _C.cuda_device_count())
        if cfg["techniques"]:
            opts["sys.techniques"] = cfg["techniques"]
        if cfg["num_channels"] != -1:
            opts["sys.channels"] = cfg["num_channels"]
        opts.update(cfg["options"])
        if options:
            opts.update(options)
        opts = {str(k): (("1" if v else "0") if isinstance(v, bool) else str(v)) for k, v in opts.items()}

        self._lens_t = None
        self._lens_dev = None
        if isinstance(value_lengths, (int, np.integer)):
            nk = num_keys if num_keys is not None else cfg["num_keys"]
            if nk is None:
                raise ValueError("num_keys is unknown: call adapm_b200.setup(num_keys, num_threads) first or pass num_keys=")
            self._impl = _C.Server(opts, int(nk), int(value_lengths), 0, 0)
            self._uniform_len = int(value_lengths)
        else:
            lt = torch.as_tensor(value_lengths).to(torch.int64).contiguous().view(-1).cpu()
            nk = num_keys if num_keys is not None else (cfg["num_keys"] if cfg["num_keys"] is not None else lt.numel())
            self._lens_t = lt
            self._impl = _C.Server(opts, int(nk), 0, lt.data_ptr(), lt.numel())
            self._uniform_len = None
        self.dtype = _DTYPES[dtype]
        self.backend = backend
        self.device = torch.device("cuda", self._impl.device()) if backend == "cuda" else torch.device("cpu")
        self._keepalive = []

    # -- sampling -----------------------------------------------------------------
    def enable_sampling_support(self, scheme: str = "local", with_replacement: bool = True,
                                distribution: str = "uniform", min: int = 0, max: int = 0,
                                weights=None, sample_fn=None) -> None:
        """Reference ``Server.enable_sampling_support`` (bindings.cc:97-135).

        ``distribution``: ``uniform`` | ``log-uniform`` over ``[min, max)``; ``weights``
        (1-D, one weight per key of ``[min, max)``) builds an alias table; ``sample_fn`` is a
        Python callable returning one key (the reference's app-provided ``Key (*)()``).
        """
        if sample_fn is not None:
            dist = _C.callback_distribution(sample_fn, int(min), int(max))
        elif weights is not None:
            w = torch.as_tensor(weights, dtype=torch.float64).contiguous().cpu()
            dist = _C.alias_distribution(w.data_ptr(), w.numel(), int(min), 1)
        elif distribution == "uniform":
            dist = _C.uniform_distribution(int(min), int(max))
        elif distribution == "log-uniform":
            dist = _C.log_uniform_distribution(int(min), int(max))
        else:
            raise ValueError(f"Unknown sampling distribution '{distribution}'")
        self._impl.enable_sampling_support(dist, scheme, 1 if with_replacement else 0)

    # -- misc ---------------------------------------------------------------------
    def barrier(self) -> None:
        self._impl.barrier()

    def allreduce_sum(self, values) -> list:
        """Sum of up to 64 floats over all ranks (collective, one call per rank, host side)."""
        return list(self._impl.allreduce_sum([float(v) for v in values]))

    def shutdown(self) -> None:
        self._impl.shutdown()

    def my_rank(self) -> int:
        return self._impl.my_rank()

    def num_servers(self) -> int:
        return self._impl.num_servers()

    def num_keys(self) -> int:
        return self._impl.num_keys()

    def get_len(self, key: int) -> int:
        return self._impl.get_len(int(key))

    def owner_of(self, key: int) -> int:
        return self._impl.owner_of(int(key))

    def is_local(self, key: int) -> bool:
        return self._impl.is_local(int(key))

    def counters(self) -> dict:
        return dict(self._impl.counters())

    def stats(self) -> str:
        return self._impl.stats_string()

    def sync_rounds(self) -> int:
        return self._impl.sync_rounds()

    def total_len(self, keys: torch.Tensor) -> int:
        if self._uniform_len is not None:
            return keys.numel() * self._uniform_len
        return int(self._lens_t[keys.cpu()].sum().item())


class Worker:
    """A logical worker bound to one server (reference ``adapm.Worker``, bindings.cc:151-371)."""

    def __init__(self, customer_id: int, server: Server) -> None:
        self.server = server
        self.customer_id = int(customer_id)
        self._impl = _C.Worker(self.customer_id, server._impl)
        self._pending = {}

    # -- helpers ------------------------------------------------------------------
    def _vals(self, vals, n_keys_t: torch.Tensor, writable: bool) -> torch.Tensor:
        if isinstance(vals, np.ndarray):
            if not vals.flags["C_CONTIGUOUS"]:
                raise ValueError("value arrays must be C-contiguous")
            vals = torch.from_numpy(vals)
        if not isinstance(vals, torch.Tensor):
            raise TypeError("vals must be a torch.Tensor or numpy.ndarray")
        if vals.dtype != self.server.dtype:
            raise TypeError(f"vals must have dtype {self.server.dtype}, got {vals.dtype}")
        if not vals.is_contiguous():
            raise ValueError("vals must be contiguous")
        return vals

    def _check(self, keys: torch.Tensor, vals: torch.Tensor) -> None:
        nk = self.server.num_keys()
        if keys.numel():
            kmax = int(keys.max().item()) if not keys.is_cuda else None
            if kmax is not None and (kmax >= nk or int(keys.min().item()) < 0):
                raise IndexError(f"At least one of the provided keys ({kmax}) is outside the key range [0, {nk})")
        if not keys.is_cuda:
            need = self.server.total_len(keys)
        elif self.server._uniform_len is None:
            need = None   # mixed lengths on the device: checked through the offsets in _io
        else:
            need = keys.numel() * self.server._uniform_len
        if need is not None and vals.numel() != need:
            raise ValueError("The provided value array does not match the size specified in the parameter server: "
                             f"{vals.numel()} != {need}")

    def _io(self, keys: torch.Tensor, vals: torch.Tensor):
        if keys.is_cuda != vals.is_cuda:
            raise ValueError("keys and vals must live on the same device type")
        if keys.is_cuda:
            if self.server.backend != "cuda":
                raise ValueError("CUDA tensors need backend='cuda'")
            offs = 0
            if self.server._uniform_len is None:
                # mixed-length store: per-key value offsets are computed on the device
                if self.server._lens_dev is None:
                    self.server._lens_dev = self.server._lens_t.to(keys.device)
                lens = self.server._lens_dev[keys]
                o = torch.cumsum(lens, 0) - lens
                if int((o[-1] + lens[-1]).item()) != vals.numel():
                    raise ValueError("The provided value array does not match the size specified in the parameter server")
                self._offs_keep = o
                offs = o.data_ptr()
            return True, torch.cuda.current_stream(keys.device).cuda_stream, offs
        return False, 0, 0

    # -- data ops -----------------------------------------------------------------
    def pull(self, keys, vals, asynchronous: bool = False) -> int:
        k = _as_keys(keys)
        v = self._vals(vals, k, True)
        self._check(k, v)
        dev, stream, offs = self._io(k, v)
        ts = self._impl.pull(k.data_ptr(), k.numel(), v.data_ptr(), dev, stream, offs)
        return self._finish(ts, asynchronous, (k, v))

    def push(self, keys, vals, asynchronous: bool = False) -> int:
        k = _as_keys(keys)
        v = self._vals(vals, k, False)
        self._check(k, v)
        dev, stream, offs = self._io(k, v)
        ts = self._impl.push(k.data_ptr(), k.numel(), v.data_ptr(), False, dev, stream, offs)
        return self._finish(ts, asynchronous, (k, v))

    def set(self, keys, vals, asynchronous: bool = False) -> int:
        k = _as_keys(keys)
        v = self._vals(vals, k, False)
        self._check(k, v)
        dev, stream, offs = self._io(k, v)
        ts = self._impl.push(k.data_ptr(), k.numel(), v.data_ptr(), True, dev, stream, offs)
        return self._finish(ts, asynchronous, (k, v))

    def _finish(self, ts: int, asynchronous: bool, keep) -> int:
        if ts == LOCAL:
            return ts
        if asynchronous:
            self._pending[ts] = keep  # caller keeps buffers alive in the reference; we do it for them
            return ts
        self._impl.wait(ts)
        return ts

    def pull_if_local(self, key: int, vals) -> bool:
        v = self._vals(vals, None, True)
        if v.is_cuda:
            tmp = torch.empty(v.shape, dtype=v.dtype)
            ok = self._impl.pull_if_local(int(key), tmp.data_ptr())
            if ok:
                v.copy_(tmp)
            return ok
        return self._impl.pull_if_local(int(key), v.data_ptr())

    # -- intent / clocks ----------------------------------------------------------
    def intent(self, keys, start: int, end: int = 0) -> int:
        k = _as_keys(keys)
        if k.is_cuda:
            k = k.cpu()
        return self._impl.intent(k.data_ptr(), k.numel(), int(start), int(end))

    def intent_fast(self, keys, start: int, end: int = 0) -> int:
        """Intent with the pre-pass on the calling thread (CPU backend): keys that already have a usable local slot
        only get their end clock extended, the others take the normal path. Returns #keys on the fast path."""
        k = _as_keys(keys)
        if k.is_cuda:
            k = k.cpu()
        return self._impl.intent_fast(k.data_ptr(), k.numel(), int(start), int(end))

    def advance_clock(self) -> int:
        return self._impl.advance_clock()

    def current_clock(self) -> int:
        return self._impl.current_clock()

    # -- sampling -----------------------------------------------------------------
    def prepare_sample(self, K: int, start: int, end: int = 0) -> int:
        return self._impl.prepare_sample(int(K), int(start), int(end))

    def pull_sample(self, sample_id: int, keys, vals, asynchronous: bool = False) -> int:
        """Fills ``keys`` (int64, output) and ``vals`` with the next ``len(keys)`` sampled keys."""
        k_out = keys
        if isinstance(keys, np.ndarray):
            k = torch.from_numpy(keys)
        else:
            k = keys
        if k.dtype != torch.int64 or not k.is_contiguous():
            raise TypeError("keys must be a contiguous int64 tensor/array (it is an output)")
        v = self._vals(vals, k, True)
        if k.is_cuda or v.is_cuda:
            kh = torch.empty(k.shape, dtype=torch.int64)
            vh = torch.empty(v.shape, dtype=v.dtype)
            ts = self._impl.pull_sample(int(sample_id), kh.data_ptr(), kh.numel(), vh.data_ptr())
            self._impl.wait(ts)
            k.copy_(kh)
            v.copy_(vh)
            return LOCAL
        ts = self._impl.pull_sample(int(sample_id), k.data_ptr(), k.numel(), v.data_ptr())
        return self._finish(ts, asynchronous, (k_out, v))

    def finish_sample(self, sample_id: int) -> None:
        self._impl.finish_sample(int(sample_id))

    # -- synchronisation ----------------------------------------------------------
    def wait(self, ts: int) -> None:
        self._impl.wait(int(ts))
        self._pending.pop(ts, None)

    def is_finished(self, ts: int) -> bool:
        return self._impl.is_finished(int(ts))

    def waitall(self) -> None:
        self._impl.wait_all()
        self._pending.clear()

    def wait_sync(self) -> None:
        self._impl.wait_sync()

    def wait_replica_sync(self) -> None:  # deprecated name kept by the reference
        self._impl.wait_sync()

    def barrier(self) -> None:
        self._impl.barrier()

    def begin_setup(self) -> None:
        self._impl.begin_setup()

    def end_setup(self) -> None:
        self._impl.end_setup()

    def finalize(self) -> None:
        self._impl.finalize()
        self._pending.clear()

    def get_key_size(self, key_id: int = 0) -> int:
        return self._impl.get_len(int(key_id))

    @property
    def num_keys(self) -> int:
        return self._impl.num_keys()

    def locality(self) -> dict:
        return dict(self._impl.locality())


__all__ = ["setup", "scheduler", "Server", "Worker", "LOCAL", "CLOCK_MAX", "AdapmError"]
