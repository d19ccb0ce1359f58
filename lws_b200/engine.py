"""ctypes binding of ``liblwse.so`` (the C ABI of ``include/lwse.h``).

This is the only way Python reaches the engine, and it is the same set of
symbols a cgo shim binds (INTEGRATION.md).  There is no fallback: if the
library is missing or no sm_90 (H100) device is present, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import records as R

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "liblwse.so")
_lib = None

# every symbol include/lwse.h declares: name → (argtypes, restype)
SYMBOLS = {
    "lwse_create": ([C.POINTER(R.Config), C.POINTER(C.c_void_p)], C.c_int),
    "lwse_destroy": ([C.c_void_p], None),
    "lwse_strerror": ([C.c_int], C.c_char_p),
    "lwse_last_cuda_error": ([C.c_void_p], C.c_int),
    "lwse_abi_version": ([], C.c_uint32),
    "lwse_stream": ([C.c_void_p], C.c_void_p),
    "lwse_launch_count": ([C.c_void_p], C.c_uint64),
    "lwse_shard_of": ([C.c_uint64, C.c_uint32], C.c_uint32),
    "lwse_hash64": ([C.c_void_p, C.c_size_t], C.c_uint64),
    "lwse_upload_nodes": ([C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32], C.c_int),
    "lwse_sweep_lws_host": ([C.c_void_p, C.POINTER(R.LwsTables)], C.c_int),
    "lwse_sweep_lws_device": ([C.c_void_p, C.POINTER(R.LwsTables), C.c_void_p], C.c_int),
    "lwse_resident_load": ([C.c_void_p, C.POINTER(R.LwsTables)], C.c_int),
    "lwse_resident_patch": ([C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_uint32], C.c_int),
    "lwse_resident_sweep": ([C.c_void_p, C.c_uint32, C.POINTER(R.Changes)], C.c_int),
    "lwse_resident_outputs": ([C.c_void_p, C.c_void_p, C.c_void_p], C.c_int),
    "lwse_resident_arena": ([C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)], C.c_int),
    "lwse_resident_place_load": ([C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32], C.c_int),
    "lwse_resident_tick": ([C.c_void_p, C.POINTER(R.Tick)], C.c_int),
    "lwse_resident_tick_submit": ([C.c_void_p, C.POINTER(R.Tick)], C.c_int),
    "lwse_resident_tick_wait": ([C.c_void_p, C.POINTER(R.Tick)], C.c_int),
    "lwse_resident_place_outputs": ([C.c_void_p, C.c_void_p], C.c_int),
    "lwse_resident_occupancy": ([C.c_void_p, C.c_void_p], C.c_int),
    "lwse_resident_tick_info": ([C.c_void_p, C.c_void_p], C.c_int),
    "lwse_resident_node_info": ([C.c_void_p, C.POINTER(R.NodeInfo)], C.c_int),
    "lwse_resident_place_whatif": ([C.c_void_p, C.POINTER(R.PlaceWhatIf)], C.c_int),
    "lwse_resident_drain_whatif": ([C.c_void_p, C.POINTER(R.DrainWhatIf)], C.c_int),
    "lwse_resident_drain_cost": ([C.c_void_p, C.c_void_p], C.c_int),
    "lwse_resident_drain_budget": ([C.c_void_p, C.POINTER(R.DrainBudgetQuery)], C.c_int),
    "lwse_resident_drain_budget_cost": ([C.c_void_p, C.c_uint32, C.c_void_p], C.c_int),
    "lwse_resident_drain_place_cost": ([C.c_void_p, C.c_uint32, C.c_void_p], C.c_int),
    "lwse_resident_drain_waves": ([C.c_void_p, C.POINTER(R.DrainWavesQuery)], C.c_int),
    "lwse_resident_ds_drain": ([C.c_void_p, C.POINTER(R.DsDrainQuery)], C.c_int),
    "lwse_resident_ds_drain_cost": ([C.c_void_p, C.c_uint32, C.c_void_p], C.c_int),
    "lwse_resident_ds_drain_waves": ([C.c_void_p, C.POINTER(R.DsDrainWavesQuery)], C.c_int),
    "lwse_resident_drain_place_waves": ([C.c_void_p, C.POINTER(R.DrainPlaceWavesQuery)], C.c_int),
    "lwse_resident_rollout_place": ([C.c_void_p, C.POINTER(R.RolloutPlaceQuery)], C.c_int),
    "lwse_resident_rollout_place_waves": ([C.c_void_p, C.POINTER(R.RolloutPlaceWavesQuery)], C.c_int),
    "lwse_resident_scale_headroom": ([C.c_void_p, C.POINTER(R.ScaleHeadroomQuery)], C.c_int),
    "lwse_resident_place_explain": ([C.c_void_p, C.POINTER(R.PlaceExplainQuery)], C.c_int),
    "lwse_place_host": (
        [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)],
        C.c_int,
    ),
    "lwse_place_device": (
        [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.c_void_p],
        C.c_int,
    ),
    "lwse_place_grouped_device": (
        [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32),
         C.POINTER(C.c_uint32), C.c_void_p],
        C.c_int,
    ),
    "lwse_place_gathered_device": (
        [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p,
         C.POINTER(C.c_uint32), C.c_void_p],
        C.c_int,
    ),
    "lwse_reconcile_device": (
        [C.c_void_p, C.POINTER(R.LwsTables), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p],
        C.c_int,
    ),
    "lwse_reconcile_host": (
        [C.c_void_p, C.POINTER(R.LwsTables), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p],
        C.c_int,
    ),
    "lwse_exchange_create": ([C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p], C.c_int),
    "lwse_exchange_connect": ([C.c_void_p, C.c_void_p], C.c_int),
    "lwse_exchange_part_bytes": ([C.c_void_p], C.c_uint64),
    "lwse_reconcile_exchanged_device": (
        [C.c_void_p, C.POINTER(R.LwsTables), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p],
        C.c_int,
    ),
    "lwse_reconcile_shared_device": (
        [C.c_void_p, C.POINTER(R.LwsTables), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p],
        C.c_int,
    ),
    "lwse_exchange_status": ([C.c_void_p, C.POINTER(C.c_uint32)], C.c_int),
    "lwse_sweep_ds_host": ([C.c_void_p, C.POINTER(R.DsTables)], C.c_int),
    "lwse_sweep_ds_device": ([C.c_void_p, C.POINTER(R.DsTables), C.c_void_p], C.c_int),
    "lwse_ds_resident_load": ([C.c_void_p, C.POINTER(R.DsTables)], C.c_int),
    "lwse_ds_resident_tick": ([C.c_void_p, C.POINTER(R.PatchSeg), C.c_uint32, C.POINTER(R.DsChanges)], C.c_int),
    "lwse_ds_resident_tick_info": ([C.c_void_p, C.POINTER(R.DsTickInfo)], C.c_int),
    "lwse_ds_forecast_host": ([C.c_void_p, C.POINTER(R.DsTables), C.POINTER(R.DsForecastOut)], C.c_int),
    "lwse_ds_resident_forecast": ([C.c_void_p, C.POINTER(R.DsForecastOut)], C.c_int),
    "lwse_resident_ds_rollout_whatif": ([C.c_void_p, C.POINTER(R.DsRolloutWhatIf)], C.c_int),
    "lwse_lws_forecast_host": (
        [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(R.LwsForecastOut)], C.c_int),
    "lwse_resident_forecast": ([C.c_void_p, C.POINTER(R.LwsForecastOut)], C.c_int),
    "lwse_resident_rollout_whatif": ([C.c_void_p, C.POINTER(R.RolloutWhatIf)], C.c_int),
    "lwse_group_keys_host": ([C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p], C.c_int),
    "lwse_subgroup_keys_host": (
        [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p], C.c_int),
    "lwse_subgroup_keys_device": (
        [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
         C.c_void_p], C.c_int),
    "lwse_group_keys_device": (
        [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p],
        C.c_int,
    ),
}


class LwseError(RuntimeError):
    def __init__(self, status: int, cuda_error: int = 0):
        self.status, self.cuda_error = status, cuda_error
        msg = lib().lwse_strerror(status).decode()
        if cuda_error:
            msg += f" [cudaError {cuda_error}]"
        super().__init__(f"lwse: {msg} ({status})")


def lib_path() -> str:
    return _LIB_PATH


def lib() -> C.CDLL:
    """Load liblwse.so; raises if it has not been built (no silent fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise FileNotFoundError(
                f"{_LIB_PATH} is missing: build it with `python -m lws_b200.build` "
                "(the engine has no CPU fallback)"
            )
        _lib = C.CDLL(_LIB_PATH)
        for name, (args, res) in SYMBOLS.items():
            fn = getattr(_lib, name)  # AttributeError = ABI drift, fail loudly
            fn.argtypes, fn.restype = args, res
    return _lib


def shard_of(uid_hash: int, n_shards: int) -> int:
    return lib().lwse_shard_of(uid_hash, n_shards)


def _aligned16(a: np.ndarray) -> np.ndarray:
    """``a`` itself when it is contiguous at a 16-byte aligned base, else an aligned copy."""
    if a.flags.c_contiguous and a.ctypes.data % 16 == 0:
        return a
    b = R.aligned_empty(len(a), a.dtype)
    b[:] = a
    return b


def rollout_waves_args(rows, ns, recs, max_waves, constraints):
    """The arguments of ``Engine.resident_rollout_place_waves`` as the call takes them → (rows, ns, recs);
    ValueError for a duplicate row, a cap outside 1 .. DRAIN_WAVES_MAX or a zero or unknown constraint bit."""
    rows = np.ascontiguousarray(rows, dtype=np.uint32)
    ns = np.ascontiguousarray(ns, dtype=np.uint32)
    if len(ns) != len(rows):
        raise ValueError("rows and ns differ in length")
    if len(np.unique(rows)) != len(rows):
        raise ValueError("rollout waves take each LWS row once")
    if not 1 <= max_waves <= R.DRAIN_WAVES_MAX:
        raise ValueError(f"max_waves must be in 1 .. {R.DRAIN_WAVES_MAX}")
    if constraints == 0 or constraints & ~R.RPW_ALL:
        raise ValueError("constraints must be a nonzero mask of RPW_* bits")
    if recs is not None:
        recs = np.asarray(recs)
        if recs.dtype != R.LWS_REC or len(recs) != len(rows):
            raise ValueError("recs must be one LWS_REC per entry")
        recs = _aligned16(recs)
    return rows, ns, recs


class Engine:
    """One engine per GPU (``lwse_create``)."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        cfg = R.Config(R.ABI_VERSION, device, 0, 0)
        rc = lib().lwse_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            raise LwseError(rc)
        self.device = device
        self.n_nodes = 0
        self.n_domains = 0

    def close(self):
        if self._h:
            lib().lwse_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise LwseError(rc, lib().lwse_last_cuda_error(self._h))

    @property
    def stream(self) -> int:
        return lib().lwse_stream(self._h) or 0

    @property
    def launch_count(self) -> int:
        return lib().lwse_launch_count(self._h)

    # ------------------------------------------------------------------ nodes
    def upload_nodes(self, nodes: np.ndarray, n_domains: int):
        assert nodes.dtype == R.NODE_REC
        self._check(lib().lwse_upload_nodes(self._h, R.ptr(nodes) if len(nodes) else None, len(nodes), n_domains))
        self.n_nodes, self.n_domains = len(nodes), n_domains

    # -------------------------------------------------------------- LWS sweep
    def sweep_lws_host(self, lws, groups, pod_state, pod_ident, flags=0, want_occupancy=False, out=None):
        """Host tables in → (lws_out, group_out, occupancy|None) host tables out."""
        assert lws.dtype == R.LWS_REC and groups.dtype == R.GROUP_REC
        assert pod_state.dtype == R.POD_STATE and pod_ident.dtype == R.POD_IDENT and len(pod_state) == len(pod_ident)
        if out is None:
            lws_out = R.aligned_empty(len(lws), R.LWS_OUT)
            group_out = R.aligned_empty(len(groups), R.GROUP_OUT)
        else:
            lws_out, group_out = out
        occ = np.zeros(max(self.n_nodes, 1), dtype=np.uint32) if want_occupancy else None
        t = R.LwsTables(
            R.ptr(lws), len(lws), R.ptr(groups), len(groups), R.ptr(pod_state), R.ptr(pod_ident), len(pod_state),
            R.ptr(lws_out), R.ptr(group_out), R.ptr(occ), flags,
        )
        self._check(lib().lwse_sweep_lws_host(self._h, C.byref(t)))
        return lws_out, group_out, (occ[: self.n_nodes] if occ is not None else None)

    def reconcile_host(self, lws, groups, pod_state, pod_ident, reqs, occupancy=None, n_namespaces=1, flags=0,
                       out=None, place_out=None):
        """Host tables + placement requests in → (lws_out, group_out, place_out): one tick, one call."""
        assert lws.dtype == R.LWS_REC and groups.dtype == R.GROUP_REC and reqs.dtype == R.PLACE_REQ
        assert pod_state.dtype == R.POD_STATE and pod_ident.dtype == R.POD_IDENT and len(pod_state) == len(pod_ident)
        lws_out, group_out = out if out is not None else (R.aligned_empty(len(lws), R.LWS_OUT),
                                                          R.aligned_empty(len(groups), R.GROUP_OUT))
        if place_out is None:
            place_out = R.aligned_empty(len(reqs), R.PLACE_OUT)
        if occupancy is not None:
            occupancy = np.ascontiguousarray(occupancy, dtype=np.uint32)
        t = R.LwsTables(
            R.ptr(lws), len(lws), R.ptr(groups), len(groups), R.ptr(pod_state), R.ptr(pod_ident), len(pod_state),
            R.ptr(lws_out), R.ptr(group_out), None, flags,
        )
        self._check(lib().lwse_reconcile_host(self._h, C.byref(t), R.ptr(reqs) if len(reqs) else None, len(reqs),
                                              R.ptr(occupancy), n_namespaces, R.ptr(place_out) if len(reqs) else None))
        return lws_out, group_out, place_out

    def sweep_lws_device(self, d_lws, n_lws, d_groups, n_groups, d_pod_state, d_pod_ident, n_pods, d_lws_out,
                         d_group_out, d_occupancy=None, flags=0, stream=None):
        """Device pointers (ints / tensors) in; kernels are enqueued, no synchronize."""
        t = R.LwsTables(
            R.ptr(d_lws), n_lws, R.ptr(d_groups), n_groups, R.ptr(d_pod_state), R.ptr(d_pod_ident), n_pods,
            R.ptr(d_lws_out), R.ptr(d_group_out), R.ptr(d_occupancy), flags,
        )
        self._check(lib().lwse_sweep_lws_device(self._h, C.byref(t), stream))

    @staticmethod
    def device_tables(d_lws, n_lws, d_groups, n_groups, d_pod_state, d_pod_ident, n_pods, d_lws_out, d_group_out,
                      d_occupancy=None, flags=0):
        """The ``lwse_lws_tables`` descriptor of device-resident tables (build once, reuse every tick)."""
        return R.LwsTables(
            R.ptr(d_lws), n_lws, R.ptr(d_groups), n_groups, R.ptr(d_pod_state), R.ptr(d_pod_ident), n_pods,
            R.ptr(d_lws_out), R.ptr(d_group_out), R.ptr(d_occupancy), flags,
        )

    def reconcile_device(self, tables, d_reqs, n_reqs, d_occupancy, n_namespaces, d_place_out, stream=None):
        """One reconcile tick: sweep on ``stream``, placement round concurrently on the engine's
        side stream, joined back into ``stream``.  Enqueue only, no synchronize."""
        self._check(lib().lwse_reconcile_device(self._h, C.byref(tables), R.ptr(d_reqs), n_reqs, R.ptr(d_occupancy),
                                                n_namespaces, R.ptr(d_place_out), stream))

    # --------------------------------------------------------- peer exchange
    def exchange_create(self, reqs_per_part: int, world: int, rank: int) -> bytes:
        """Allocate this rank's exchange buffer → its 64-byte IPC handle (all-gather these)."""
        h = (C.c_uint8 * 64)()
        self._check(lib().lwse_exchange_create(self._h, reqs_per_part, world, rank, h))
        return bytes(h)

    def exchange_connect(self, handles: bytes):
        """``handles``: every rank's handle, concatenated in rank order."""
        buf = (C.c_uint8 * len(handles)).from_buffer_copy(handles)
        self._check(lib().lwse_exchange_connect(self._h, buf))

    @property
    def exchange_part_bytes(self) -> int:
        return int(lib().lwse_exchange_part_bytes(self._h))

    def reconcile_exchanged_device(self, tables, d_local_part, n_namespaces, d_place_out, stream=None):
        """One tick of a shard: push this rank's [occupancy | requests] part to every peer over
        NVLink, wait for theirs, placement round over all parts — on the side stream, concurrently
        with the sweep of ``tables`` (None: placement step only).  Enqueue only."""
        self._check(lib().lwse_reconcile_exchanged_device(
            self._h, C.byref(tables) if tables is not None else None, R.ptr(d_local_part), n_namespaces,
            R.ptr(d_place_out), stream))

    def reconcile_shared_device(self, tables, d_reqs, n_reqs, d_local_occupancy, n_namespaces, d_place_out, flags=0, stream=None):
        """One tick of a shard with LOCAL requests and SHARED occupancy: the rank's occupancy counters go to
        every peer over NVLink, the local (namespace-grouped) requests are solved against the sum — on the
        side stream, concurrently with the sweep of ``tables`` (None: placement branch only)."""
        self._check(lib().lwse_reconcile_shared_device(
            self._h, C.byref(tables) if tables is not None else None, R.ptr(d_reqs), n_reqs, R.ptr(d_local_occupancy),
            n_namespaces, R.ptr(d_place_out), flags, stream))

    def exchange_status(self) -> int:
        err = C.c_uint32(0)
        self._check(lib().lwse_exchange_status(self._h, C.byref(err)))
        return err.value

    # ------------------------------------------------------- resident tables
    def resident_load(self, lws, groups, pod_state, pod_ident):
        """Make the four input tables resident on the device."""
        self._resident_shape = (len(lws), len(groups))
        self._resident_pods = len(pod_state)
        self._n_place = 0
        t = R.LwsTables(R.ptr(lws), len(lws), R.ptr(groups), len(groups), R.ptr(pod_state), R.ptr(pod_ident),
                        len(pod_state), None, None, None, 0)
        self._check(lib().lwse_resident_load(self._h, C.byref(t)))
        self._chg = None

    _DT = {R.TABLE_LWS: R.LWS_REC, R.TABLE_GROUPS: R.GROUP_REC, R.TABLE_POD_STATE: R.POD_STATE,
           R.TABLE_POD_IDENT: R.POD_IDENT, R.TABLE_PLACE_REQS: R.PLACE_REQ, R.TABLE_NODES: R.NODE_REC}

    # ----------------------------------------------------------- resident tick
    def resident_arena(self, min_bytes: int = 0) -> np.ndarray:
        """The engine's pinned, mapped patch arena as a uint8 array: patch rows / values written
        into it are read by the GPU in place (no staging copy)."""
        base, size = C.c_void_p(), C.c_uint64()
        self._check(lib().lwse_resident_arena(self._h, min_bytes, C.byref(base), C.byref(size)))
        buf = (C.c_uint8 * size.value).from_address(base.value)
        return np.frombuffer(buf, dtype=np.uint8)

    def resident_place_load(self, reqs: np.ndarray, n_namespaces: int = 1):
        assert reqs.dtype == R.PLACE_REQ
        self._n_place = len(reqs)
        self._check(lib().lwse_resident_place_load(self._h, R.ptr(reqs) if len(reqs) else None, len(reqs), n_namespaces))

    def make_tick(self, segments=(), flags=0) -> "R.Tick":
        """Build a reusable ``lwse_tick`` descriptor.  ``segments``: (table, rows, values) with
        numpy arrays (ideally views of the arena), or (table, first_row, values, True) for a range."""
        segs = (R.PatchSeg * max(len(segments), 1))()
        keep = []
        for i, sg in enumerate(segments):
            if len(sg) == 4 and sg[3]:
                table, first, values = sg[0], sg[1], sg[2]
                segs[i] = R.PatchSeg(table, R.PATCH_RANGE, len(values), int(first), None, R.ptr(values))
                keep.append(values)
            else:
                table, rows, values = sg[0], sg[1], sg[2]
                assert rows.dtype == np.uint32 and len(rows) == len(values) and values.dtype == self._DT[table]
                segs[i] = R.PatchSeg(table, 0, len(rows), 0, R.ptr(rows) if len(rows) else None,
                                     R.ptr(values) if len(rows) else None)
                keep.append((rows, values))
        t = R.Tick()
        t.segs = segs
        t.n_segs = len(segments)
        t.flags = flags
        t._keep = (segs, keep)
        return t

    def resident_tick(self, tick: "R.Tick"):
        """One tick: patches in, changed result rows out (views of engine-owned pinned memory,
        valid until the next resident call).  → dict of numpy views."""
        self._check(lib().lwse_resident_tick(self._h, C.byref(tick)))
        return self._tick_views(tick)

    def resident_tick_submit(self, tick: "R.Tick"):
        """Enqueue a tick and return (at most two in flight); its patch segments stay untouched in the
        arena until the matching ``resident_tick_wait``."""
        self._check(lib().lwse_resident_tick_submit(self._h, C.byref(tick)))

    def resident_tick_wait(self, tick: "R.Tick" = None):
        """Wait for the OLDEST submitted tick → the same dict as ``resident_tick`` (views valid until
        the second submit after this call)."""
        tick = tick if tick is not None else R.Tick()
        self._check(lib().lwse_resident_tick_wait(self._h, C.byref(tick)))
        return self._tick_views(tick)

    def _tick_views(self, tick: "R.Tick"):
        def view(ptr, n, dtype):
            if not ptr or n == 0:
                return np.zeros(0, dtype=dtype)
            nbytes = n * np.dtype(dtype).itemsize
            return np.frombuffer((C.c_uint8 * nbytes).from_address(ptr), dtype=dtype)

        n_lws = min(tick.n_lws, self._resident_shape[0])
        n_grp = min(tick.n_groups, self._resident_shape[1])
        n_pl = min(tick.n_place, getattr(self, "_n_place", 0))
        return {
            "lws_rows": view(tick.lws_rows, n_lws, np.uint32), "lws_out": view(tick.lws_out, n_lws, R.LWS_OUT),
            "group_rows": view(tick.group_rows, n_grp, np.uint32), "group_out": view(tick.group_out, n_grp, R.GROUP_OUT),
            "place_rows": view(tick.place_rows, n_pl, np.uint32), "place_out": view(tick.place_out, n_pl, R.PLACE_OUT),
            "n_lws": tick.n_lws, "n_groups": tick.n_groups, "n_place": tick.n_place, "rounds": tick.place_rounds,
        }

    def resident_place_outputs(self) -> np.ndarray:
        out = R.aligned_empty(self._n_place, R.PLACE_OUT)
        self._check(lib().lwse_resident_place_outputs(self._h, R.ptr(out)))
        return out

    def resident_occupancy(self) -> np.ndarray:
        occ = np.zeros(max(self.n_nodes, 1), dtype=np.uint32)
        self._check(lib().lwse_resident_occupancy(self._h, R.ptr(occ)))
        return occ[: self.n_nodes]

    TICK_FORMS = {0: "none", 1: "general", 2: "namespace", 3: "scan"}

    def resident_tick_info(self) -> dict:
        """How the most recently submitted tick ran: ``form`` (none | general | namespace | scan),
        ``indexed`` (the namespace form went through the namespace index: the request table is not
        grouped), ``index_built`` (this tick rebuilt that index), ``graph`` (replayed as a CUDA graph)."""
        w = (C.c_uint32 * 4)()
        self._check(lib().lwse_resident_tick_info(self._h, w))
        return {"form": self.TICK_FORMS[w[0]], "indexed": bool(w[1]), "index_built": bool(w[2]), "graph": bool(w[3])}

    def resident_node_info(self) -> dict:
        """What the node-row patches of the most recently submitted tick did: ``rows_patched``,
        ``index_built`` (its placement round rebuilt the domain-sorted node index first: a patch changed
        whether a node is usable, or a usable node's domain) and ``n_usable`` (usable nodes after it)."""
        info = R.NodeInfo()
        self._check(lib().lwse_resident_node_info(self._h, C.byref(info)))
        return {"rows_patched": info.rows_patched, "index_built": bool(info.index_built), "n_usable": info.n_usable}

    def resident_place_whatif(self, segs=(), extra=None, n_namespaces=0, capacity=None):
        """lwse_resident_place_whatif: the placement round over the resident tables with ``segs`` (NODES and
        PLACE_REQS segments, as ``make_tick`` takes them) applied and the ``extra`` request rows appended —
        nothing resident changes, and no tick is waited for.  ``capacity`` None lists every changed row.
        → dict: ``rows`` / ``before`` / ``after`` (the resident rows that differ from the last round, with
        both rows), ``extra_out`` (the rows of the extra requests), the counters of ``records.PLACE_WHATIF``
        and ``form`` (namespace | general)."""
        tick = self.make_tick(segs)
        n_res = getattr(self, "_n_place", 0)
        extra = R.aligned_empty(0, R.PLACE_REQ) if extra is None else _aligned16(np.asarray(extra, dtype=R.PLACE_REQ))
        cap = n_res if capacity is None else int(capacity)
        rows = np.zeros(max(cap, 1), np.uint32)
        before, after = R.aligned_empty(max(cap, 1), R.PLACE_OUT), R.aligned_empty(max(cap, 1), R.PLACE_OUT)
        extra_out = R.aligned_empty(max(len(extra), 1), R.PLACE_OUT)
        q = R.PlaceWhatIf()
        q.segs = C.cast(tick.segs, C.c_void_p) if len(segs) else None
        q.n_segs = len(segs)
        q.extra = R.ptr(extra) if len(extra) else None
        q.n_extra = len(extra)
        q.n_namespaces = int(n_namespaces)
        q.capacity = cap
        q.rows, q.before, q.after = R.ptr(rows), R.ptr(before), R.ptr(after)
        q.extra_out = R.ptr(extra_out) if len(extra) else None
        self._check(lib().lwse_resident_place_whatif(self._h, C.byref(q)))
        n = min(q.n_changed, cap)
        out = {"rows": rows[:n], "before": before[:n], "after": after[:n], "extra_out": extra_out[: len(extra)],
               "form": self.TICK_FORMS[q.form]}
        out.update({k: getattr(q, k) for k in R.PLACE_WHATIF})
        return out

    def resident_place_explain(self, rows=None, mask=R.PLACE_UNSCHEDULABLE | R.PLACE_CONFLICT, segs=(), extra=None,
                               n_namespaces=0, capacity=None):
        """lwse_resident_place_explain: why rows of a placement round have their verdicts.  The round is the
        baseline (the last tick's rows) without ``segs``, ``extra`` and a new ``n_namespaces``, else the what-if
        round ``resident_place_whatif`` computes for them.  ``rows`` lists row indices into the round; None takes
        every row whose result flags share a bit with ``mask`` (``records.PLACE_*``), ascending.  ``capacity`` None
        returns every explained row.  → dict: ``rows`` (``records.PLACE_EXPLAIN``), ``n_explained``,
        ``round_rows``, ``n_domains``, ``whatif``, ``form``, ``classes`` ({class: sum over the rows}) and ``flags``
        ({``records.PEX_NAMES`` name: rows carrying it}).  Changes nothing resident and waits for no tick."""
        tick = self.make_tick(segs)
        extra = R.aligned_empty(0, R.PLACE_REQ) if extra is None else _aligned16(np.asarray(extra, dtype=R.PLACE_REQ))
        listed = None if rows is None else np.ascontiguousarray(rows, dtype=np.uint32)
        buf = None if listed is None else (listed if len(listed) else np.zeros(1, np.uint32))  # (non-NULL: a list)
        bound = (getattr(self, "_n_place", 0) + len(extra)) if listed is None else len(listed)
        cap = bound if capacity is None else int(capacity)
        out = R.aligned_empty(max(cap, 1), R.PLACE_EXPLAIN)
        q = R.PlaceExplainQuery()
        q.segs = C.cast(tick.segs, C.c_void_p) if len(segs) else None
        q.n_segs = len(segs)
        q.extra = R.ptr(extra) if len(extra) else None
        q.n_extra = len(extra)
        q.n_namespaces = int(n_namespaces)
        q.mask = int(mask)
        q.rows = R.ptr(buf)
        q.n_rows = 0 if listed is None else len(listed)
        q.capacity = cap
        q.out = R.ptr(out)
        self._check(lib().lwse_resident_place_explain(self._h, C.byref(q)))
        res = {"rows": out[: min(q.n_explained, cap)], "n_explained": q.n_explained, "round_rows": q.round_rows,
               "n_domains": q.n_domains, "whatif": bool(q.whatif),
               "form": self.TICK_FORMS[q.form] if q.whatif else None}
        res["classes"] = {k: int(q.n_class[j]) for j, k in enumerate(R.PLACE_EXPLAIN_CLASSES)}
        res["flags"] = {name: int(q.n_flag[b.bit_length() - 1]) for b, name in R.PEX_NAMES.items()}
        return res

    def resident_drain_whatif(self, nodes, capacity=None):
        """lwse_resident_drain_whatif: the group rows of a sweep of the resident tables with every pod scheduled
        on one of the node rows ``nodes`` (and every leader whose group row names one) deleting — nothing
        resident changes, and no tick is waited for.  ``capacity`` None lists every changed row.
        → dict: ``rows`` / ``before`` / ``after`` (the group rows that differ from the last sweep, with both
        rows) and the counters of ``records.DRAIN_WHATIF``."""
        nodes = np.ascontiguousarray(nodes, dtype=np.uint32)
        n_res = getattr(self, "_resident_shape", (0, 0))[1]
        cap = n_res if capacity is None else int(capacity)
        rows = np.zeros(max(cap, 1), np.uint32)
        before, after = R.aligned_empty(max(cap, 1), R.GROUP_OUT), R.aligned_empty(max(cap, 1), R.GROUP_OUT)
        q = R.DrainWhatIf()
        q.nodes = R.ptr(nodes) if len(nodes) else None
        q.n_nodes = len(nodes)
        q.capacity = cap
        q.rows, q.before, q.after = R.ptr(rows), R.ptr(before), R.ptr(after)
        self._check(lib().lwse_resident_drain_whatif(self._h, C.byref(q)))
        n = min(q.n_changed, cap)
        out = {"rows": rows[:n], "before": before[:n], "after": after[:n]}
        out.update({k: getattr(q, k) for k in R.DRAIN_WHATIF})
        return out

    def resident_drain_cost(self) -> np.ndarray:
        """lwse_resident_drain_cost: one ``records.DRAIN_COST`` row per node of the resident node table, row n
        holding the counters ``resident_drain_whatif([n])`` returns — every node in one pass."""
        out = R.aligned_empty(max(self.n_nodes, 1), R.DRAIN_COST)
        self._check(lib().lwse_resident_drain_cost(self._h, R.ptr(out)))
        return out[: self.n_nodes]

    _DRAIN_SCOPES = {"nodes": R.DRAIN_NODES, "domains": R.DRAIN_DOMAINS}

    @staticmethod
    def _drain_ids(nodes, domains):
        """A drain set given as exactly one of node rows or domain ids → (ids as uint32, its ``records.DRAIN_*``
        scope)."""
        if (nodes is None) == (domains is None):
            raise ValueError("give node rows or domain ids")
        ids = np.ascontiguousarray(nodes if domains is None else domains, dtype=np.uint32)
        return ids, R.DRAIN_NODES if domains is None else R.DRAIN_DOMAINS

    def _drain_waves(self, call, query, key_dtype, wave_dtype, totals, nodes, domains, max_waves, constraints=None):
        """One waves plan: a ``query`` filled and passed to ``call`` → dict: the key rows, the opened wave rows and
        the fields ``totals`` names."""
        ids, scope = self._drain_ids(nodes, domains)
        keys = R.aligned_empty(max(len(ids), 1), key_dtype)
        waves = R.aligned_empty(max(int(max_waves), 1), wave_dtype)
        q = query()
        q.ids = R.ptr(ids) if len(ids) else None
        q.n_ids = len(ids)
        q.scope = scope
        q.max_waves = int(max_waves)
        if constraints is not None:
            q.constraints = int(constraints)
        q.keys, q.waves = R.ptr(keys), R.ptr(waves)
        self._check(call(self._h, C.byref(q)))
        out = {"keys": keys[: len(ids)], "waves": waves[: q.n_waves]}
        out.update({k: getattr(q, k) for k in totals})
        return out

    def resident_drain_budget(self, nodes=None, domains=None, capacity=None):
        """lwse_resident_drain_budget: the LeaderWorkerSet rows a drain of the node rows ``nodes`` — or of every
        node in the domain ids ``domains`` — touches, each with its availability floor, ready count before
        and after, and ``records.DRAINB_*`` flags.  Give exactly one of the two.  ``capacity`` None lists every
        touched row.  → dict: ``rows`` (``records.DRAIN_BUDGET``) and the totals of
        ``records.DRAIN_BUDGET_TOTALS``."""
        ids, scope = self._drain_ids(nodes, domains)
        n_res = getattr(self, "_resident_shape", (0, 0))[0]
        cap = n_res if capacity is None else int(capacity)
        rows = R.aligned_empty(max(cap, 1), R.DRAIN_BUDGET)
        q = R.DrainBudgetQuery()
        q.ids = R.ptr(ids) if len(ids) else None
        q.n_ids = len(ids)
        q.scope = scope
        q.capacity = cap
        q.rows = R.ptr(rows)
        self._check(lib().lwse_resident_drain_budget(self._h, C.byref(q)))
        out = {"rows": rows[: min(q.n_touched, cap)]}
        out.update({k: getattr(q, k) for k in R.DRAIN_BUDGET_TOTALS})
        return out

    def resident_drain_budget_cost(self, scope: str = "nodes") -> np.ndarray:
        """lwse_resident_drain_budget_cost: one ``records.DRAIN_BUDGET_COST`` row per node (``scope="nodes"``) or
        per domain (``"domains"``), row k holding the answer ``resident_drain_budget`` gives for that key alone
        — every key in one call."""
        n = self.n_nodes if scope == "nodes" else self.n_domains
        out = R.aligned_empty(max(n, 1), R.DRAIN_BUDGET_COST)
        self._check(lib().lwse_resident_drain_budget_cost(self._h, self._DRAIN_SCOPES[scope], R.ptr(out)))
        return out[:n]

    def resident_drain_waves(self, nodes=None, domains=None, max_waves=R.DRAIN_WAVES_MAX):
        """lwse_resident_drain_waves: the distinct node rows ``nodes`` — or domain ids ``domains`` — packed first-fit,
        in the order given, into at most ``max_waves`` waves whose drain takes no LeaderWorkerSet below its
        floor.  Give exactly one of the two.  → dict: ``keys`` (``records.DRAIN_WAVE_KEY``, in query order),
        ``waves`` (``records.DRAIN_WAVE``, one per opened wave) and the totals of ``records.DRAIN_WAVES_TOTALS``."""
        return self._drain_waves(lib().lwse_resident_drain_waves, R.DrainWavesQuery, R.DRAIN_WAVE_KEY, R.DRAIN_WAVE,
                                 R.DRAIN_WAVES_TOTALS, nodes, domains, max_waves)

    def resident_drain_place_cost(self, scope: str = "nodes") -> np.ndarray:
        """lwse_resident_drain_place_cost: one ``records.DRAIN_PLACE_COST`` row per node (``scope="nodes"``) or per
        domain (``"domains"``), row k holding what the three calls ``resident_drain_whatif`` →
        ``IncrementalEncoder.drain_place_query`` → ``resident_place_whatif`` answer for that key alone: whether
        the groups the drain restarts find a new exclusive domain — every key in one call."""
        n = self.n_nodes if scope == "nodes" else self.n_domains
        out = R.aligned_empty(max(n, 1), R.DRAIN_PLACE_COST)
        self._check(lib().lwse_resident_drain_place_cost(self._h, self._DRAIN_SCOPES[scope], R.ptr(out)))
        return out[:n]

    def resident_ds_drain(self, nodes=None, domains=None, capacity=None, outputs=False):
        """lwse_resident_ds_drain: the DisaggregatedSets a drain of the node rows ``nodes`` — or of every node in
        the domain ids ``domains`` — touches through their linked child LeaderWorkerSets, each with its
        ``records.DSD_*`` verdicts and its ds_out row in the before and the after sweep.  Give exactly one of the
        two.  ``capacity`` None lists every touched DS; ``outputs`` also returns the after sweep's full
        ``role_out`` / ``revrole_out``.  → dict: ``rows`` (``records.DS_DRAIN``) and the totals of
        ``records.DS_DRAIN_TOTALS``."""
        ids, scope = self._drain_ids(nodes, domains)
        n_ds, n_roles, n_rr = getattr(self, "_ds_shape", (0, 0, 0))
        cap = n_ds if capacity is None else int(capacity)
        rows = R.aligned_empty(max(cap, 1), R.DS_DRAIN)
        q = R.DsDrainQuery()
        q.ids = R.ptr(ids) if len(ids) else None
        q.n_ids = len(ids)
        q.scope = scope
        q.capacity = cap
        q.rows = R.ptr(rows)
        role_out = revrole_out = None
        if outputs:
            role_out = R.aligned_empty(max(n_roles, 1), R.DS_ROLE_OUT)
            revrole_out = R.aligned_empty(max(n_rr, 1), R.DS_REVROLE_OUT)
            q.role_out, q.revrole_out = R.ptr(role_out), R.ptr(revrole_out)
        self._check(lib().lwse_resident_ds_drain(self._h, C.byref(q)))
        out = {"rows": rows[: min(q.n_touched, cap)]}
        out.update({k: getattr(q, k) for k in R.DS_DRAIN_TOTALS})
        if outputs:
            out["role_out"], out["revrole_out"] = role_out[:n_roles], revrole_out[:n_rr]
        return out

    def resident_ds_drain_cost(self, scope: str = "nodes") -> np.ndarray:
        """lwse_resident_ds_drain_cost: one ``records.DS_DRAIN_COST`` row per node (``scope="nodes"``) or per
        domain (``"domains"``), row k holding the counts ``resident_ds_drain`` gives for that key alone — every
        key in one call."""
        n = self.n_nodes if scope == "nodes" else self.n_domains
        out = R.aligned_empty(max(n, 1), R.DS_DRAIN_COST)
        self._check(lib().lwse_resident_ds_drain_cost(self._h, self._DRAIN_SCOPES[scope], R.ptr(out)))
        return out[:n]

    def resident_ds_drain_waves(self, nodes=None, domains=None, max_waves=R.DRAIN_WAVES_MAX,
                                constraints=R.DSW_LWS_FLOOR | R.DSW_DS_SERVICE | R.DSW_DS_OLD_SERVICE):
        """lwse_resident_ds_drain_waves: the distinct node rows ``nodes`` — or domain ids ``domains`` — packed
        first-fit, in the order given, into at most ``max_waves`` waves whose drain triggers none of the verdicts
        in ``constraints`` (``records.DSW_*``).  The default keeps every LeaderWorkerSet at its floor and every
        DisaggregatedSet serving; ``DSW_DS_STALL`` is opt-in, since it forbids any ready loss under a rolling DS.
        Give exactly one of the two.  → dict: ``keys`` (``records.DS_DRAIN_WAVE_KEY``, in query order), ``waves``
        (``records.DS_DRAIN_WAVE``, one per opened wave) and the totals of ``records.DS_DRAIN_WAVES_TOTALS``."""
        return self._drain_waves(lib().lwse_resident_ds_drain_waves, R.DsDrainWavesQuery, R.DS_DRAIN_WAVE_KEY,
                                 R.DS_DRAIN_WAVE, R.DS_DRAIN_WAVES_TOTALS, nodes, domains, max_waves, constraints)

    def resident_drain_place_waves(self, nodes=None, domains=None, max_waves=R.DRAIN_WAVES_MAX,
                                   constraints=R.DPW_LWS_FLOOR | R.DPW_STRANDED):
        """lwse_resident_drain_place_waves: the distinct node rows ``nodes`` — or domain ids ``domains`` — packed
        first-fit, in the order given, into at most ``max_waves`` waves whose drain triggers none of the verdicts in
        ``constraints`` (``records.DPW_*``).  The default keeps every LeaderWorkerSet at its floor and finds every
        request the wave unpins a new exclusive domain; ``DPW_BUMPED`` (no other request loses its domain) is
        opt-in.  Give exactly one of the two.  → dict: ``keys`` (``records.DRAIN_PLACE_WAVE_KEY``, in query order),
        ``waves`` (``records.DRAIN_PLACE_WAVE``, one per opened wave) and the totals of
        ``records.DRAIN_WAVES_TOTALS``."""
        return self._drain_waves(lib().lwse_resident_drain_place_waves, R.DrainPlaceWavesQuery, R.DRAIN_PLACE_WAVE_KEY,
                                 R.DRAIN_PLACE_WAVE, R.DRAIN_WAVES_TOTALS, nodes, domains, max_waves, constraints)

    def resident_patch(self, which: int, rows, values):
        """Overwrite rows of a resident table (rows: uint32 indices, values: packed rows)."""
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        values = np.ascontiguousarray(values, dtype=self._DT[which])
        assert len(rows) == len(values)
        self._check(lib().lwse_resident_patch(self._h, which, R.ptr(rows) if len(rows) else None,
                                              R.ptr(values) if len(rows) else None, len(rows)))

    def resident_sweep(self, flags=0, lws_capacity=None, group_capacity=None):
        """Sweep the resident tables → (lws_rows, lws_out, group_rows, group_out, n_lws_changed,
        n_groups_changed): only result rows that changed since the previous resident sweep."""
        n_lws, n_grp = self._resident_shape
        lc = n_lws if lws_capacity is None else lws_capacity
        gc = n_grp if group_capacity is None else group_capacity
        if self._chg is None or self._chg[0] != (lc, gc):
            self._chg = ((lc, gc), np.zeros(max(lc, 1), np.uint32), R.aligned_empty(max(lc, 1), R.LWS_OUT),
                         np.zeros(max(gc, 1), np.uint32), R.aligned_empty(max(gc, 1), R.GROUP_OUT))
        _, lr, lo, gr, go = self._chg
        ch = R.Changes(R.ptr(lr), R.ptr(lo), lc, 0, R.ptr(gr), R.ptr(go), gc, 0)
        self._check(lib().lwse_resident_sweep(self._h, flags, C.byref(ch)))
        nl, ng = min(ch.n_lws, lc), min(ch.n_groups, gc)
        return lr[:nl], lo[:nl], gr[:ng], go[:ng], ch.n_lws, ch.n_groups

    def resident_outputs(self):
        n_lws, n_grp = self._resident_shape
        lo, go = R.aligned_empty(n_lws, R.LWS_OUT), R.aligned_empty(n_grp, R.GROUP_OUT)
        self._check(lib().lwse_resident_outputs(self._h, R.ptr(lo), R.ptr(go)))
        return lo, go

    # -------------------------------------------------------------- placement
    def place_host(self, reqs: np.ndarray, occupancy=None, n_namespaces=1):
        assert reqs.dtype == R.PLACE_REQ
        out = R.aligned_empty(len(reqs), R.PLACE_OUT)
        rounds = C.c_uint32(0)
        if occupancy is not None:
            occupancy = np.ascontiguousarray(occupancy, dtype=np.uint32)
        self._check(
            lib().lwse_place_host(self._h, R.ptr(reqs), len(reqs), R.ptr(occupancy), n_namespaces,
                                  R.ptr(out), C.byref(rounds))
        )
        return out, rounds.value

    def place_device(self, d_reqs, n_reqs, d_occupancy, n_namespaces, d_out, stream=None, want_rounds=False):
        """Enqueue a placement round; synchronizes only when ``want_rounds``."""
        rounds = C.c_uint32(0)
        self._check(
            lib().lwse_place_device(self._h, R.ptr(d_reqs), n_reqs, R.ptr(d_occupancy), n_namespaces,
                                    R.ptr(d_out), C.byref(rounds) if want_rounds else None, stream)
        )
        return rounds.value if want_rounds else None

    def place_grouped_device(self, d_reqs, n_reqs, d_occupancy, n_namespaces, d_out, flags=0, stream=None, want_rounds=False):
        """Placement round over a request table grouped by namespace (one CTA per namespace; flags:
        SWEEP_PLACE_SCAN = brute-force (request x node) form).  → (rounds, scans) when ``want_rounds``."""
        rounds, scans = C.c_uint32(0), C.c_uint32(0)
        self._check(lib().lwse_place_grouped_device(self._h, R.ptr(d_reqs), n_reqs, R.ptr(d_occupancy), n_namespaces,
                                                    R.ptr(d_out), flags, C.byref(rounds) if want_rounds else None,
                                                    C.byref(scans) if want_rounds else None, stream))
        return (rounds.value, scans.value) if want_rounds else None

    def place_gathered_device(self, d_parts, n_parts, part_stride_bytes, reqs_offset_bytes, reqs_per_part,
                              n_namespaces, d_out, stream=None, want_rounds=False):
        """Placement over the all-gathered [occupancy | requests] parts of every rank."""
        rounds = C.c_uint32(0)
        self._check(
            lib().lwse_place_gathered_device(self._h, R.ptr(d_parts), n_parts, part_stride_bytes, reqs_offset_bytes,
                                             reqs_per_part, n_namespaces, R.ptr(d_out),
                                             C.byref(rounds) if want_rounds else None, stream)
        )
        return rounds.value if want_rounds else None

    # --------------------------------------------------------------------- DS
    def sweep_ds_host(self, ds, roles, revroles, out=None):
        """lwse_sweep_ds_host: host tables in, host result rows out.  `out` = (ds_out, role_out, revrole_out)
        arrays to fill instead of fresh ones (page-locked tables and outputs copy at PCIe speed; pageable ones
        are staged by the driver)."""
        assert ds.dtype == R.DS_REC and roles.dtype == R.DS_ROLE_REC and revroles.dtype == R.DS_REVROLE_REC
        if out is None:
            ds_out = R.aligned_empty(len(ds), R.DS_OUT)
            role_out = R.aligned_empty(len(roles), R.DS_ROLE_OUT)
            revrole_out = R.aligned_empty(len(revroles), R.DS_REVROLE_OUT)
        else:
            ds_out, role_out, revrole_out = out
            assert ds_out.dtype == R.DS_OUT and role_out.dtype == R.DS_ROLE_OUT and revrole_out.dtype == R.DS_REVROLE_OUT
            assert len(ds_out) == len(ds) and len(role_out) == len(roles) and len(revrole_out) == len(revroles)
        t = R.DsTables(
            R.ptr(ds), len(ds), R.ptr(roles), len(roles), R.ptr(revroles), len(revroles),
            R.ptr(ds_out), R.ptr(role_out), R.ptr(revrole_out),
        )
        self._check(lib().lwse_sweep_ds_host(self._h, C.byref(t)))
        return ds_out, role_out, revrole_out

    def sweep_ds_device(self, d_ds, n_ds, d_roles, n_roles, d_revroles, n_revroles, d_ds_out, d_role_out,
                        d_revrole_out, stream=None):
        t = R.DsTables(
            R.ptr(d_ds), n_ds, R.ptr(d_roles), n_roles, R.ptr(d_revroles), n_revroles,
            R.ptr(d_ds_out), R.ptr(d_role_out), R.ptr(d_revrole_out),
        )
        self._check(lib().lwse_sweep_ds_device(self._h, C.byref(t), stream))

    # ------------------------------------------------------------ resident DS
    _DS_DT = {R.TABLE_DS: R.DS_REC, R.TABLE_DS_ROLES: R.DS_ROLE_REC, R.TABLE_DS_REVROLES: R.DS_REVROLE_REC}

    def ds_resident_load(self, ds, roles, revroles):
        """Make the three DS input tables resident (sizes fixed until the next load; the next tick lists
        every DS).  Never waits for the LeaderWorkerSet ticks in flight."""
        assert ds.dtype == R.DS_REC and roles.dtype == R.DS_ROLE_REC and revroles.dtype == R.DS_REVROLE_REC
        t = R.DsTables(R.ptr(ds) if len(ds) else None, len(ds), R.ptr(roles) if len(roles) else None, len(roles),
                       R.ptr(revroles) if len(revroles) else None, len(revroles), None, None, None)
        self._check(lib().lwse_ds_resident_load(self._h, C.byref(t)))
        self._ds_shape = (len(ds), len(roles), len(revroles))

    def ds_resident_tick(self, segments=()):
        """One DS tick: ``segments`` as for ``make_tick`` ((table, rows, values), or (table, first_row,
        values, True) for a range) of the tables TABLE_DS / TABLE_DS_ROLES / TABLE_DS_REVROLES /
        TABLE_DS_LINKS; rows and values may live anywhere in host memory.  Once a link patch arrived
        (since the DS load), linked revision-role rows read their child's ready count from the
        resident LWS results of the most recently submitted LWS tick (lwse.h, ``lwse_ds_link``).
        → dict: ``rows`` (the DS rows whose decisions changed) and ``ds_out`` / ``role_out`` /
        ``revrole_out``, views of the FULL output tables kept current in engine-owned pinned memory
        (valid until the next DS call)."""
        segs = (R.PatchSeg * max(len(segments), 1))()
        keep = []
        for i, sg in enumerate(segments):
            if len(sg) == 4 and sg[3]:
                table, first, values = sg[0], sg[1], np.ascontiguousarray(sg[2])
                segs[i] = R.PatchSeg(table, R.PATCH_RANGE, len(values), int(first), None,
                                     R.ptr(values) if len(values) else None)
                keep.append(values)
            else:
                table, rows, values = sg[0], np.ascontiguousarray(sg[1], dtype=np.uint32), np.ascontiguousarray(sg[2])
                assert len(rows) == len(values) and values.dtype == self._DS_DT.get(table, values.dtype)
                segs[i] = R.PatchSeg(table, 0, len(rows), 0, R.ptr(rows) if len(rows) else None,
                                     R.ptr(values) if len(rows) else None)
                keep.append((rows, values))
        ch = R.DsChanges()
        self._check(lib().lwse_ds_resident_tick(self._h, segs, len(segments), C.byref(ch)))
        n_ds, n_roles, n_rr = self._ds_shape

        def view(ptr, n, dtype):
            if not ptr or n == 0:
                return np.zeros(0, dtype=dtype)
            return np.frombuffer((C.c_uint8 * (n * np.dtype(dtype).itemsize)).from_address(ptr), dtype=dtype)

        return {"rows": view(ch.ds_rows, min(ch.n_changed, n_ds), np.uint32), "n_changed": ch.n_changed,
                "ds_out": view(ch.ds_out, n_ds, R.DS_OUT), "role_out": view(ch.role_out, n_roles, R.DS_ROLE_OUT),
                "revrole_out": view(ch.revrole_out, n_rr, R.DS_REVROLE_OUT)}

    def ds_resident_tick_info(self) -> dict:
        """How the last DS tick read ready counts: ``linked`` (it ran the linked sweep),
        ``rows_from_lws`` (existing revision-role rows that took the LWS tick's value),
        ``rows_fallback`` (linked rows that used their own ready count) and ``lws_ticks`` (LWS ticks
        submitted when it read the LWS rows)."""
        info = R.DsTickInfo()
        self._check(lib().lwse_ds_resident_tick_info(self._h, C.byref(info)))
        return {"linked": bool(info.linked), "rows_from_lws": info.rows_from_lws,
                "rows_fallback": info.rows_fallback, "lws_ticks": info.lws_ticks}

    # ------------------------------------------------------- rollout forecast
    def _ds_forecast(self, call, n_ds, n_roles, steps, step_capacity):
        fc = R.aligned_empty(n_ds, R.DS_FORECAST)
        fr = R.aligned_empty(n_roles, R.DS_FORECAST_ROLE)
        traj = None
        if steps:
            if step_capacity is None:  # every DS's rows fit: at most the cycle cap per DS (sized by a first pass)
                probe = R.DsForecastOut(R.ptr(fc) if n_ds else None, R.ptr(fr) if n_roles else None, None, 0, 0, 0)
                self._check(call(probe))
                step_capacity = int(probe.n_steps_needed)
            traj = R.aligned_empty(max(int(step_capacity), 1), R.DS_ROLE_OUT)
        out = R.DsForecastOut(R.ptr(fc) if n_ds else None, R.ptr(fr) if n_roles else None,
                              R.ptr(traj) if traj is not None else None, int(step_capacity or 0), 0, 0)
        self._check(call(out))
        return {"ds": fc, "roles": fr, "steps": traj[: out.n_steps_written] if traj is not None else None,
                "n_steps_written": out.n_steps_written, "n_steps_needed": out.n_steps_needed}

    def ds_forecast_host(self, ds, roles, revroles, steps=True, step_capacity=None):
        """lwse_ds_forecast_host: the rest of every DS rollout, replayed from these host tables with
        every child ready before each cycle (lwse.h, "rollout forecast").  → dict: ``ds`` (DS_FORECAST
        per DS), ``roles`` (DS_FORECAST_ROLE per role row), ``steps`` (DS_ROLE_OUT {old, new} trajectory
        rows, DS d's at ``ds[d]["step_base"]``; None when ``steps`` is False), ``n_steps_written``,
        ``n_steps_needed``.  ``step_capacity`` None sizes the buffer so that every trajectory fits: it
        runs a summaries-only call first (a second summary pass) to learn the rows needed; callers
        that forecast repeatedly pass a capacity instead."""
        assert ds.dtype == R.DS_REC and roles.dtype == R.DS_ROLE_REC and revroles.dtype == R.DS_REVROLE_REC
        t = R.DsTables(R.ptr(ds) if len(ds) else None, len(ds), R.ptr(roles) if len(roles) else None, len(roles),
                       R.ptr(revroles) if len(revroles) else None, len(revroles), None, None, None)
        return self._ds_forecast(lambda o: lib().lwse_ds_forecast_host(self._h, C.byref(t), C.byref(o)),
                                 len(ds), len(roles), steps, step_capacity)

    def ds_resident_forecast(self, steps=True, step_capacity=None):
        """lwse_ds_resident_forecast: as ``ds_forecast_host`` over the resident DS tables as the last DS
        tick left them.  Changes no DS tick output and never waits for the LeaderWorkerSet ticks."""
        n_ds, n_roles, _ = getattr(self, "_ds_shape", (0, 0, 0))
        return self._ds_forecast(lambda o: lib().lwse_ds_resident_forecast(self._h, C.byref(o)),
                                 n_ds, n_roles, steps, step_capacity)

    def resident_ds_rollout_whatif(self, proposals, roles=None, steps=True, step_capacity=None):
        """lwse_resident_ds_rollout_whatif: for each proposal (DS_PROPOSAL: a resident DS row and DSP_* flags)
        the DS controller's first decision over the rows the edit would encode to (``now``, DS_OUT, and
        ``now_roles``, DS_ROLE_OUT, DS_MAX_ROLES rows per proposal) and the forecast of the rollout it would
        start, each as if it were the only edit (lwse.h, "DS rollout what-if").  ``roles``: DS_ROLE_REC rows,
        DS_MAX_ROLES per proposal (an (n, DS_MAX_ROLES) or flat array), read for DSP_ROLES proposals.  → ``now``,
        ``now_roles`` plus what ``ds_resident_forecast`` returns, with one ``ds`` row and DS_MAX_ROLES ``roles``
        rows per proposal and the trajectory offsets running over the proposals in order.  Changes nothing
        resident and waits for no tick."""
        props = np.ascontiguousarray(proposals)
        assert props.dtype == R.DS_PROPOSAL
        n, nr = len(props), len(props) * R.DS_MAX_ROLES
        if roles is not None:
            roles = np.asarray(roles).reshape(-1)
            assert roles.dtype == R.DS_ROLE_REC and len(roles) == nr
            roles = _aligned16(roles)
        now = R.aligned_empty(n, R.DS_OUT)
        now_roles = R.aligned_empty(nr, R.DS_ROLE_OUT)

        def call(o):
            q = R.DsRolloutWhatIf(R.ptr(props) if n else None, R.ptr(roles) if roles is not None and n else None, n, 0,
                                  R.ptr(now) if n else None, R.ptr(now_roles) if n else None, o)
            rc = lib().lwse_resident_ds_rollout_whatif(self._h, C.byref(q))
            o.n_steps_written, o.n_steps_needed = q.fc.n_steps_written, q.fc.n_steps_needed
            return rc

        out = self._ds_forecast(call, n, nr, steps, step_capacity)
        out["now"], out["now_roles"] = now, now_roles
        return out

    # ------------------------------------------- rolling-update forecast (LWS)
    def _lws_forecast(self, call, n_lws, steps, step_capacity):
        fc = R.aligned_empty(n_lws, R.LWS_FORECAST)
        traj = None
        if steps:
            if step_capacity is None:  # every object's rows fit (sized by a summaries-only call)
                probe = R.LwsForecastOut(R.ptr(fc) if n_lws else None, None, 0, 0, 0)
                self._check(call(probe))
                step_capacity = int(probe.n_steps_needed)
            traj = R.aligned_empty(max(int(step_capacity), 1), R.LWS_FORECAST_STEP)
        out = R.LwsForecastOut(R.ptr(fc) if n_lws else None, R.ptr(traj) if traj is not None else None,
                               int(step_capacity or 0), 0, 0)
        self._check(call(out))
        return {"lws": fc, "steps": traj[: out.n_steps_written] if traj is not None else None,
                "n_steps_written": out.n_steps_written, "n_steps_needed": out.n_steps_needed}

    def lws_forecast(self, lws, group_out, steps=True, step_capacity=None):
        """lwse_lws_forecast_host: the rest of every LeaderWorkerSet rolling update, replayed from these
        object rows and the group result rows of a sweep of the same tables (lwse.h, "rolling-update
        forecast").  → dict: ``lws`` (LWS_FORECAST per object), ``steps`` (LWS_FORECAST_STEP trajectory
        rows, object i's at ``lws[i]["step_base"]``; None when ``steps`` is False), ``n_steps_written``,
        ``n_steps_needed``.  ``step_capacity`` None sizes the buffer so that every trajectory fits, with
        a summaries-only call first; callers that forecast repeatedly pass a capacity instead."""
        assert lws.dtype == R.LWS_REC and group_out.dtype == R.GROUP_OUT
        lws, group_out = _aligned16(lws), _aligned16(group_out)
        return self._lws_forecast(
            lambda o: lib().lwse_lws_forecast_host(self._h, R.ptr(lws) if len(lws) else None, len(lws),
                                                   R.ptr(group_out) if len(group_out) else None, len(group_out),
                                                   C.byref(o)),
            len(lws), steps, step_capacity)

    def resident_forecast(self, steps=True, step_capacity=None):
        """lwse_resident_forecast: as ``lws_forecast`` over the resident LWS rows and the group results of
        the most recently submitted sweep, in flight or not; waits for no tick and changes none.  Raises
        (NOT_READY) before a sweep after a load, or after LWS / group / pod patches made without one."""
        n_lws = getattr(self, "_resident_shape", (0, 0))[0]
        return self._lws_forecast(lambda o: lib().lwse_resident_forecast(self._h, C.byref(o)), n_lws, steps,
                                  step_capacity)

    def resident_rollout_whatif(self, rows, recs, steps=True, step_capacity=None):
        """lwse_resident_rollout_whatif: for each proposal (resident row ``rows[i]``, proposed LWS_REC
        ``recs[i]``), the controller's first write (``now``, LWS_OUT) and the forecast of the rollout it
        would start, each as if it were the only edit (lwse.h, "rollout what-if").  The proposals'
        group_base / group_count are taken from the resident rows.  → ``now`` plus what
        ``resident_forecast`` returns, with one ``lws`` row per proposal and the trajectory offsets running
        over the proposals in order.  Changes nothing resident and waits for no tick."""
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        recs = np.asarray(recs)
        assert recs.dtype == R.LWS_REC and len(recs) == len(rows)
        recs = _aligned16(recs)
        now = R.aligned_empty(len(rows), R.LWS_OUT)
        n = len(rows)

        def call(o):
            q = R.RolloutWhatIf(R.ptr(rows) if n else None, R.ptr(recs) if n else None, n, 0,
                                R.ptr(now) if n else None, o)
            rc = lib().lwse_resident_rollout_whatif(self._h, C.byref(q))
            o.n_steps_written, o.n_steps_needed = q.fc.n_steps_written, q.fc.n_steps_needed
            return rc

        out = self._lws_forecast(call, n, steps, step_capacity)
        out["now"] = now
        return out

    def resident_rollout_place(self, rows, ns, recs=None, extra=False):
        """lwse_resident_rollout_place: for each entry (resident LWS row ``rows[i]``, namespace id ``ns[i]`` and,
        with ``recs``, a proposed LWS_REC as ``resident_rollout_whatif`` takes it), whether the groups its rollout
        adds up to the forecast's peak find an exclusive domain — each entry answered on its own, as the
        composition ``resident_forecast`` (or ``resident_rollout_whatif``) → extra request rows →
        ``resident_place_whatif`` would (lwse.h, "rollout placement").  → dict: ``rows`` (``records.ROLLOUT_PLACE``,
        one per entry), the query's ``lws_rows`` and ``ns``, the totals of ``records.ROLLOUT_PLACE_TOTALS`` and,
        with ``extra``, ``extra``: every entry's extra request rows (PLACE_REQ), entry after entry in query order.  Changes nothing resident and waits
        for no tick."""
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        ns = np.ascontiguousarray(ns, dtype=np.uint32)
        assert len(ns) == len(rows)
        n = len(rows)
        if recs is not None:
            recs = np.asarray(recs)
            assert recs.dtype == R.LWS_REC and len(recs) == n
            recs = _aligned16(recs)
        out = R.aligned_empty(max(n, 1), R.ROLLOUT_PLACE)
        q = R.RolloutPlaceQuery()
        q.rows = R.ptr(rows) if n else None
        q.ns = R.ptr(ns) if n else None
        q.recs = R.ptr(recs) if (recs is not None and n) else None
        q.n = n
        q.out = R.ptr(out)
        if extra:  # sized by a first call without them
            probe = R.RolloutPlaceQuery.from_buffer_copy(q)
            self._check(lib().lwse_resident_rollout_place(self._h, C.byref(probe)))
            xs = R.aligned_empty(max(probe.n_surge, 1), R.PLACE_REQ)
            q.extra, q.extra_capacity = R.ptr(xs), probe.n_surge
        self._check(lib().lwse_resident_rollout_place(self._h, C.byref(q)))
        res = {"rows": out[:n], "lws_rows": rows, "ns": ns}
        res.update({k: getattr(q, k) for k in R.ROLLOUT_PLACE_TOTALS})
        if extra:
            res["extra"] = xs[: min(q.n_surge, probe.n_surge)]
        return res

    def resident_rollout_place_waves(self, rows, ns, recs=None, max_waves=R.DRAIN_WAVES_MAX,
                                     constraints=R.RPW_STRANDED, alone=False):
        """lwse_resident_rollout_place_waves: the entries of ``resident_rollout_place`` (distinct ``rows``) packed
        first-fit, in the order given, into at most ``max_waves`` waves whose rollouts, pushed together, trigger
        none of the verdicts in ``constraints`` (``records.RPW_*``).  The default finds every group the wave's
        rollouts add an exclusive domain; ``RPW_BUMPED`` (no resident group loses its domain) is opt-in.  → dict:
        ``keys`` (``records.ROLLOUT_WAVE_KEY``, in query order), ``waves`` (``records.ROLLOUT_WAVE``, one per opened
        wave), the query's ``lws_rows`` and ``ns``, the totals of ``records.ROLLOUT_WAVES_TOTALS`` and, with
        ``alone``, ``alone_rows``: ``resident_rollout_place``'s rows for the same query.  Changes nothing resident
        and waits for no tick."""
        rows, ns, recs = rollout_waves_args(rows, ns, recs, max_waves, constraints)
        n = len(rows)
        keys = R.aligned_empty(max(n, 1), R.ROLLOUT_WAVE_KEY)
        waves = R.aligned_empty(max_waves, R.ROLLOUT_WAVE)
        q = R.RolloutPlaceWavesQuery()
        q.rows = R.ptr(rows) if n else None
        q.ns = R.ptr(ns) if n else None
        q.recs = R.ptr(recs) if (recs is not None and n) else None
        q.n, q.max_waves, q.constraints = n, max_waves, constraints
        q.keys, q.waves = R.ptr(keys), R.ptr(waves)
        if alone:
            alone_rows = R.aligned_empty(max(n, 1), R.ROLLOUT_PLACE)
            q.alone_rows = R.ptr(alone_rows)
        self._check(lib().lwse_resident_rollout_place_waves(self._h, C.byref(q)))
        res = {"keys": keys[:n], "waves": waves[: q.n_waves], "lws_rows": rows, "ns": ns}
        res.update({k: getattr(q, k) for k in R.ROLLOUT_WAVES_TOTALS})
        if alone:
            res["alone_rows"] = alone_rows[:n]
        return res

    def resident_scale_headroom(self, rows, ns, ceilings=None, constraints=R.RPW_STRANDED, current=False):
        """lwse_resident_scale_headroom: for each entry (resident LWS row ``rows[i]``, namespace id ``ns[i]`` and,
        with ``ceilings``, a ceiling such as an HPA's maxReplicas, negative for none), the largest replicas the
        object can scale to before a group it adds triggers a verdict of ``constraints`` (``records.RPW_*``,
        ``RPW_STRANDED`` always included) — answered for settled exclusive objects (lwse.h, "scale headroom").
        → dict: ``rows`` (``records.SCALE_HEADROOM``, one per entry), the query's ``lws_rows``, ``ns`` and
        ``ceilings``, the totals of ``records.SCALE_HEADROOM_TOTALS`` and, with ``current``, ``current``:
        ``resident_rollout_place``'s rows of the resident rows.  Changes nothing resident and waits for no tick."""
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        ns = np.ascontiguousarray(ns, dtype=np.uint32)
        if len(ns) != len(rows):
            raise ValueError("rows and ns differ in length")
        n = len(rows)
        if ceilings is not None:
            ceilings = np.ascontiguousarray(ceilings, dtype=np.int32)
            if len(ceilings) != n:
                raise ValueError("ceilings must be one int32 per entry")
        out = R.aligned_empty(max(n, 1), R.SCALE_HEADROOM)
        q = R.ScaleHeadroomQuery()
        q.rows = R.ptr(rows) if n else None
        q.ns = R.ptr(ns) if n else None
        q.ceilings = R.ptr(ceilings) if (ceilings is not None and n) else None
        q.n, q.constraints = n, constraints
        q.out = R.ptr(out)
        if current:
            cur = R.aligned_empty(max(n, 1), R.ROLLOUT_PLACE)
            q.current = R.ptr(cur)
        self._check(lib().lwse_resident_scale_headroom(self._h, C.byref(q)))
        res = {"rows": out[:n], "lws_rows": rows, "ns": ns, "ceilings": ceilings}
        res.update({k: getattr(q, k) for k in R.SCALE_HEADROOM_TOTALS})
        if current:
            res["current"] = cur[:n]
        return res

    # ------------------------------------------------------------- group keys
    def group_keys_host(self, strings) -> np.ndarray:
        """SHA-1 of each string → (n, 20) uint8."""
        enc = [s.encode() if isinstance(s, str) else bytes(s) for s in strings]
        offsets = np.zeros(len(enc) + 1, dtype=np.uint32)
        offsets[1:] = np.cumsum([len(b) for b in enc], dtype=np.uint64).astype(np.uint32)
        blob = np.frombuffer(b"".join(enc) + b"\0", dtype=np.uint8)
        digests = np.zeros((len(enc), 20), dtype=np.uint8)
        self._check(
            lib().lwse_group_keys_host(self._h, R.ptr(blob), R.ptr(offsets), len(enc), R.ptr(digests))
        )
        return digests

    def subgroup_keys_host(self, leader_names, pod_count, subgroup_size, worker_index):
        """getSubGroupIndex + SHA-1("<leaderName>/<index>") for a batch of pods → (index int32[n], digests (n, 20))."""
        enc = [s.encode() if isinstance(s, str) else bytes(s) for s in leader_names]
        n = len(enc)
        offsets = np.zeros(n + 1, dtype=np.uint32)
        offsets[1:] = np.cumsum([len(b) for b in enc], dtype=np.uint64).astype(np.uint32)
        blob = np.frombuffer(b"".join(enc) + b"\0\0\0\0", dtype=np.uint8)
        pc, sg, wi = (np.ascontiguousarray(x, dtype=np.int32) for x in (pod_count, subgroup_size, worker_index))
        index = np.zeros(n, dtype=np.int32)
        digests = np.zeros((n, 20), dtype=np.uint8)
        self._check(lib().lwse_subgroup_keys_host(self._h, R.ptr(blob), R.ptr(offsets), n, R.ptr(pc), R.ptr(sg), R.ptr(wi),
                                                  R.ptr(index), R.ptr(digests)))
        return index, digests

    def group_keys_device(self, d_bytes, d_offsets, n, d_digests, stream=None):
        self._check(lib().lwse_group_keys_device(self._h, R.ptr(d_bytes), R.ptr(d_offsets), n, R.ptr(d_digests), stream))
