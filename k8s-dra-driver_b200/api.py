"""ctypes binding of libdra_alloc.so (include/dra_alloc.h) — the same entry points a Go driver binds
with cgo (INTEGRATION.md).  This module is plumbing: every call below crosses the C ABI and runs the
sm_90a kernels; nothing is computed in Python and nothing falls back to the CPU.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import records as R

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libdra_alloc.so")

OK, E_INVAL, E_CUDA, E_NCCL, E_NOMEM, E_STATE = 0, -1, -2, -3, -4, -5
CFG_USE_GRAPH, CFG_NO_FUSED, CFG_NO_DIRECT, CFG_RESIDENT = 0x1, 0x2, 0x4, 0x8
F_NODE_SORTED, F_FRESH_INVENTORY, F_EXHAUSTIVE = 0x1, 0x2, 0x4
PRE_FITS, PRE_EVICT, PRE_NO, PRE_SEARCH_LIMIT, PRE_INVALID = 0, 1, 2, 3, 4     # dra_preempt_batch statuses (spec §14)
PDB_NONE = 0xFFFFFFFF                                                           # a running pod under no disruption budget
# DRA_K_*: the kernels an Allocate-family call enqueued (dra_debug_last_chain)
KERNELS = {"fused_staged": 0x00001, "fused_stream": 0x00002, "fused_direct": 0x00004, "serve": 0x00008,
           "sorted_prep": 0x00010, "bucket_small": 0x00020, "hist8": 0x00040, "hist8_multi": 0x00080,
           "hist_warp": 0x00100, "scan8": 0x00200, "scan_rows": 0x00400, "scan": 0x00800, "scatter": 0x01000,
           "pack1": 0x02000, "pack4": 0x04000, "compact_flat1": 0x08000, "compact_flat8": 0x10000,
           "compact_lookback": 0x20000, "compact_in_kernel": 0x40000, "pod_shard": 0x80000, "pod_gather": 0x100000, "place": 0x200000,
           "place_shard": 0x400000, "preempt": 0x800000, "preempt_shard": 0x1000000,
           "preempt_place": 0x2000000, "preempt_place_shard": 0x4000000, "pod_capacity": 0x8000000,
           "pod_capacity_shard": 0x10000000}


class DraError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libdra_alloc: rc={code}: {msg}")
        self.code = code


class _Cfg(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("device", C.c_int32), ("stream", C.c_void_p),
                ("max_claims", C.c_uint32), ("flags", C.c_uint32)]


class RunningPods(C.Structure):
    """dra_running_pods: the running pods of dra_preempt_batch (spec §14)."""
    _fields_ = [("claims", C.c_void_p), ("n_claim", C.c_uint32), ("pod_off", C.c_void_p), ("n_pod", C.c_uint32),
                ("prio", C.c_void_p), ("out_off", C.c_void_p), ("out", C.c_void_p), ("n_out", C.c_uint32)]


class DisruptionBudgets(C.Structure):
    """dra_disruption_budgets: the budget of each running pod (PDB_NONE for none) and each budget's disruptionsAllowed."""
    _fields_ = [("run_pdb", C.c_void_p), ("allowed", C.c_void_p), ("n_pdb", C.c_uint32)]


# every symbol include/dra_alloc.h declares: name -> (restype, argtypes)
_vp, _u32, _i32, _u64 = C.c_void_p, C.c_uint32, C.c_int, C.c_uint64
SYMBOLS = {
    "dra_abi_version": (_i32, []),
    "dra_ctx_create": (_i32, [C.POINTER(_Cfg), C.POINTER(_vp)]),
    "dra_ctx_destroy": (None, [_vp]),
    "dra_last_error": (C.c_char_p, [_vp]),
    "dra_set_placement_table": (_i32, [_vp, _u32, _vp]),
    "dra_set_inventory": (_i32, [_vp, _vp, _u32, _vp, _u32]),
    "dra_set_gpu_attrs": (_i32, [_vp, _vp, _u32]),
    "dra_set_selectors": (_i32, [_vp, _vp, _u32]),
    "dra_get_inventory": (_i32, [_vp, _vp, _u32]),
    "dra_reset_inventory": (_i32, [_vp]),
    "dra_allocate_batch": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _u32]),
    "dra_allocate_batch_device": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _u32]),
    "dra_ctx_sync": (_i32, [_vp]),
    "dra_unsuitable_batch": (_i32, [_vp, _vp, _u32, _vp, _u32, _vp, _vp, _vp, _u32]),
    "dra_allocate_pods_batch": (_i32, [_vp, _vp, _u32, _vp, _u32, _vp, _vp, _u32, _u32]),
    "dra_place_pods_batch": (_i32, [_vp, _vp, _u32, _vp, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _u32]),
    "dra_deallocate_batch": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32]),
    "dra_preempt_batch": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32]),
    "dra_preempt_pdb_batch": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                     _u32, _u32]),
    "dra_preempt_place_batch": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _u32, _vp, _vp, _vp, _u32]),
    "dra_pod_capacity_batch": (_i32, [_vp, _vp, _u32, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _u32]),
    "dra_comm_unique_id": (_i32, [_vp]),
    "dra_comm_init": (_i32, [_vp, _vp, _i32, _i32]),
    "dra_allocate_batch_gather_device": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _u32, _u32]),
    "dra_gather_table": (_i32, [_vp, C.POINTER(_vp), C.POINTER(_u32)]),
    "dra_gather_read": (_i32, [_vp, _vp, _u32]),
    "dra_peer_export": (_i32, [_vp, _u32, _vp]),
    "dra_peer_import": (_i32, [_vp, _vp]),
    "dra_comm_init_local": (_i32, [_vp, _i32, _i32]),
    "dra_peer_import_local": (_i32, [_vp, _vp]),
    "dra_peer_rendezvous_device": (_i32, [_vp]),
    "dra_set_shard": (_i32, [_vp, _u32, _u32, _i32]),
    "dra_set_shard_map": (_i32, [_vp, _vp, _i32]),
    "dra_shard_export": (_i32, [_vp, _u32, _u32, _vp]),
    "dra_allocate_batch_global_device": (_i32, [_vp, _vp, _u32, _vp, _u32, _u32]),
    "dra_set_shard_pairs": (_i32, [_vp, _u32]),
    "dra_unsuitable_batch_global_device": (_i32, [_vp, _vp, _u32, _vp, _u32, _vp, _vp, _u32, _vp, _u32]),
    "dra_allocate_pods_batch_global_device": (_i32, [_vp, _vp, _u32, _vp, _u32, _vp, _u32, _u32]),
    "dra_set_shard_place": (_i32, [_vp, _u32]),
    "dra_place_pods_batch_global_device": (_i32, [_vp, _vp, _u32, _vp, _u32, _vp, _vp, _u32, _vp, _u32, _vp, _u32]),
    "dra_set_shard_preempt": (_i32, [_vp, _u32, _u32, _u32]),
    "dra_preempt_batch_global_device": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp,
                                               _vp, _u32, _u32]),
    "dra_preempt_pdb_batch_global_device": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp,
                                                   _vp, _vp, _vp, _vp, _vp, _u32, _u32]),
    "dra_set_shard_preempt_place": (_i32, [_vp, _u32, _u32, _u32]),
    "dra_preempt_place_batch_global_device": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp,
                                                     _vp, _u32]),
    "dra_set_shard_capacity": (_i32, [_vp, _u32]),
    "dra_pod_capacity_batch_global_device": (_i32, [_vp, _vp, _u32, _vp, _u32, _vp, _vp, _u32, _u32, _vp, _vp, _vp, _vp,
                                                    _u32]),
    "dra_shard_sync_inventory_device": (_i32, [_vp]),
    "dra_deallocate_batch_global_device": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32]),
    "dra_mps_limits_batch": (_i32, [_vp, _vp, _u32, _vp, _vp]),
    "dra_imex_offsets_batch": (_i32, [_vp, _vp, _vp, _u32, C.c_int32, C.c_int32, _vp]),
    "dra_calibrate": (_i32, [_vp, C.POINTER(_u32)]),
    "dra_serve_start": (_i32, [_vp]),
    "dra_serve_stop": (_i32, [_vp]),
    "dra_serve_batches": (_u64, [_vp]),
    "dra_host_alloc": (_vp, [C.c_size_t]),
    "dra_host_free": (None, [_vp]),
    "dra_launch_count": (_u64, [_vp]),
    "dra_set_profiling": (_i32, [_vp, _i32]),
    "dra_debug_timeline": (_i32, [_vp, _vp, _u32]),
    "dra_debug_last_chain": (_i32, [_vp, C.POINTER(_u32), C.POINTER(_u32)]),
    "dra_debug_shard_times": (_i32, [_vp, _vp]),
    "dra_debug_serve_times": (_i32, [_vp, _vp]),
    "dra_debug_noop": (_i32, [_vp, _u32, _u32, _u32]),
    "dra_get_timings": (_i32, [_vp, _vp, _i32]),
}

_lib = None


def load(build_if_stale: bool = True) -> C.CDLL:
    """dlopen the in-tree library; raises if it is missing — there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_stale:
        from . import build as _b
        try:
            if _b.stale():
                _b.build()
        except RuntimeError:
            if not os.path.exists(SO_PATH):
                raise
    if not os.path.exists(SO_PATH):
        raise FileNotFoundError(f"{SO_PATH} not built: run `python __graft_entry__.py build`; "
                                "the allocation path has no CPU fallback")
    lib = C.CDLL(SO_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError if the ABI and the header drift apart
        fn.restype, fn.argtypes = res, args
    if lib.dra_abi_version() != 2:
        raise RuntimeError("libdra_alloc ABI version mismatch")
    _lib = lib
    return lib


def _cands(cand_nodes, cand_off):
    """(cand_nodes, cand_off) as the C calls take them: both None in the dense form, else uint32 arrays with an empty
    cand_nodes made one element long, since NULL would mean the dense form."""
    if cand_nodes is None and cand_off is None:
        return None, None
    cn = np.ascontiguousarray(cand_nodes if cand_nodes is not None else [], dtype=np.uint32)
    return (cn if len(cn) else np.zeros(1, np.uint32)), np.ascontiguousarray(cand_off, dtype=np.uint32)


def _running(claims, pod_off, prio, out, out_off=None) -> RunningPods:
    """RunningPods over contiguous copies of the arrays, which it keeps alive."""
    keep = (np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE), np.ascontiguousarray(pod_off, dtype=np.uint32),
            np.ascontiguousarray(prio, dtype=np.int32), np.ascontiguousarray(out, dtype=R.OUT_DTYPE),
            None if out_off is None else np.ascontiguousarray(out_off, dtype=np.uint32))
    c, po, pr, o, oo = keep
    run = RunningPods(c.ctypes.data, len(c), po.ctypes.data, len(po) - 1, pr.ctypes.data,
                      None if oo is None else oo.ctypes.data, o.ctypes.data, len(o))
    run._keep = keep
    return run


def _placed_n_out(claims, out_off) -> int:
    """n_out for claims whose node is still to be chosen: their slots as if every claim named a node of the inventory."""
    if out_off is None:
        return len(claims)
    placed = claims.copy()
    placed["node"] = 0
    return int(R.claim_slots(placed, 1).sum())


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    return a.ctypes.data_as(C.c_void_p)


class PinnedBuffer:
    """Page-locked host array from dra_host_alloc: passing it to Context calls skips staging."""

    def __init__(self, n: int, dtype):
        self._lib = load()
        dtype = np.dtype(dtype)
        self.nbytes = max(16, int(n) * dtype.itemsize)
        self.ptr = self._lib.dra_host_alloc(self.nbytes)
        if not self.ptr:
            raise MemoryError("dra_host_alloc failed")
        buf = (C.c_uint8 * self.nbytes).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(n))

    def free(self):
        if self.ptr:
            self.array = None
            self._lib.dra_host_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Context:
    """One dra_ctx: one CUDA device, one stream, one inventory."""

    def __init__(self, device: int = 0, stream: int | None = None, max_claims: int = 0, flags: int = 0):
        self._lib = load()
        cfg = _Cfg(2, device, C.c_void_p(stream) if stream else None, max_claims, flags)
        h = C.c_void_p()
        rc = self._lib.dra_ctx_create(C.byref(cfg), C.byref(h))
        if rc != OK:
            raise DraError(rc, (self._lib.dra_last_error(None) or b"").decode())
        self._h = h
        self.n_gpu = 0
        self.n_node = 0

    # -- plumbing -----------------------------------------------------------------------------------
    def _check(self, rc: int):
        if rc != OK:
            raise DraError(rc, (self._lib.dra_last_error(self._h) or b"").decode())

    def close(self):
        if getattr(self, "_h", None):
            self._lib.dra_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # -- state ----------------------------------------------------------------------------------------
    def set_table(self, table: np.ndarray):
        """table: PROF_DTYPE[MAX_MODELS, MAX_PROFILES]"""
        t = np.ascontiguousarray(table, dtype=R.PROF_DTYPE)
        assert t.shape == (R.MAX_MODELS, R.MAX_PROFILES)
        for m in range(R.MAX_MODELS):
            self._check(self._lib.dra_set_placement_table(self._h, m, _ptr(t[m])))

    def set_inventory(self, gpus: np.ndarray, node_off: np.ndarray):
        g = np.ascontiguousarray(gpus, dtype=R.GPU_DTYPE)
        off = np.ascontiguousarray(node_off, dtype=np.uint32)
        self._check(self._lib.dra_set_inventory(self._h, _ptr(g), len(g), _ptr(off), len(off) - 1))
        self.n_gpu, self.n_node = len(g), len(off) - 1

    def set_gpu_attrs(self, attrs: np.ndarray | None):
        if attrs is None or len(attrs) == 0:
            self._check(self._lib.dra_set_gpu_attrs(self._h, None, 0))
            return
        a = np.ascontiguousarray(attrs, dtype=R.ATTR_DTYPE)
        self._check(self._lib.dra_set_gpu_attrs(self._h, _ptr(a), len(a)))

    def set_selectors(self, sels: np.ndarray | None):
        if sels is None or len(sels) == 0:
            self._check(self._lib.dra_set_selectors(self._h, None, 0))
            return
        s_ = np.ascontiguousarray(sels, dtype=R.SEL_INS_DTYPE).reshape(-1, R.SEL_MAX_INS)
        self._check(self._lib.dra_set_selectors(self._h, _ptr(s_), len(s_)))

    def get_inventory(self) -> np.ndarray:
        g = np.zeros(self.n_gpu, dtype=R.GPU_DTYPE)
        self._check(self._lib.dra_get_inventory(self._h, _ptr(g), self.n_gpu))
        return g

    def reset_inventory(self):
        self._check(self._lib.dra_reset_inventory(self._h))

    def sync(self):
        self._check(self._lib.dra_ctx_sync(self._h))

    # -- the path ---------------------------------------------------------------------------------------
    def allocate(self, claims: np.ndarray, out_off: np.ndarray | None = None, n_out: int | None = None,
                 flags: int = 0, out: np.ndarray | None = None) -> np.ndarray:
        c = claims if (claims.dtype == R.CLAIM_DTYPE and claims.flags.c_contiguous) else \
            np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
        oo = None if out_off is None else np.ascontiguousarray(out_off, dtype=np.uint32)
        if n_out is None:
            n_out = len(c) if oo is None else int(R.claim_slots(c, self.n_node).sum())
        if out is None:
            out = np.zeros(n_out, dtype=R.OUT_DTYPE)
        self._check(self._lib.dra_allocate_batch(self._h, _ptr(c), len(c), _ptr(oo), _ptr(out), n_out, flags))
        return out

    def allocate_raw(self, claims_ptr: int, n_claim: int, out_off_ptr: int | None, out_ptr: int, n_out: int,
                     flags: int = 0) -> None:
        """dra_allocate_batch on raw HOST addresses (e.g. PinnedBuffer.ptr): the bare C-ABI call, without the
        numpy conveniences of allocate() — what a cgo caller pays."""
        rc = self._lib.dra_allocate_batch(self._h, claims_ptr, n_claim, out_off_ptr, out_ptr, n_out, flags)
        if rc != OK:
            self._check(rc)

    def allocate_device(self, d_claims: int, n_claim: int, d_out_off: int | None, d_out: int, n_out: int,
                        flags: int = 0):
        """Device pointers (ints); enqueues on the context's stream, no synchronisation."""
        self._check(self._lib.dra_allocate_batch_device(self._h, _ptr(d_claims), n_claim, _ptr(d_out_off),
                                                        _ptr(d_out), n_out, flags))

    def allocate_gather_device(self, d_claims: int, n_claim: int, d_out_off: int | None, d_out_all: int,
                               n_out: int, n_per_rank: int, flags: int = 0):
        self._check(self._lib.dra_allocate_batch_gather_device(self._h, _ptr(d_claims), n_claim,
                                                               _ptr(d_out_off), _ptr(d_out_all), n_out,
                                                               n_per_rank, flags))

    def allocate_pods(self, claims, pod_off, out_off=None, n_out=None, flags: int = 0) -> np.ndarray:
        """Pod mode (spec §12): every pod atomically; flags & F_EXHAUSTIVE = backtracking placement search."""
        c = np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
        po = np.ascontiguousarray(pod_off, dtype=np.uint32)
        oo = None if out_off is None else np.ascontiguousarray(out_off, dtype=np.uint32)
        if n_out is None:
            n_out = len(c) if oo is None else int(R.claim_slots(c, self.n_node).sum())
        out = np.zeros(n_out, dtype=R.OUT_DTYPE)
        self._check(self._lib.dra_allocate_pods_batch(self._h, _ptr(c), len(c), _ptr(po), len(po) - 1, _ptr(oo), _ptr(out),
                                                      n_out, flags))
        return out

    def place_pods(self, claims, pod_off, cand_nodes=None, cand_off=None, out_off=None, n_out=None, flags: int = 0):
        """Choose the node and allocate (spec §13): pods in input order, each on its first candidate where it fits given
        what the pods before it took.  cand_nodes/cand_off None = every node, ascending.  The claims' node fields are
        ignored.  Returns (out, pod_node); pod_node[p] = 0xFFFFFFFF when the pod was placed nowhere.
        flags: F_EXHAUSTIVE, F_FRESH_INVENTORY."""
        c = np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
        po = np.ascontiguousarray(pod_off, dtype=np.uint32)
        oo = None if out_off is None else np.ascontiguousarray(out_off, dtype=np.uint32)
        if n_out is None:
            n_out = _placed_n_out(c, oo)
        cn, co = _cands(cand_nodes, cand_off)
        n_pod = len(po) - 1
        out = np.zeros(n_out, dtype=R.OUT_DTYPE)
        pod_node = np.zeros(max(n_pod, 1), dtype=np.uint32)
        self._check(self._lib.dra_place_pods_batch(self._h, _ptr(c), len(c), _ptr(po), n_pod, _ptr(cn), _ptr(co), _ptr(oo),
                                                   _ptr(out), n_out, _ptr(pod_node), flags))
        return out, pod_node[:n_pod]

    def unsuitable(self, claims, pod_off, cand_nodes=None, cand_off=None, flags: int = 0) -> np.ndarray:
        """cand_nodes/cand_off None = dense form: every pod against every node (bit k = pod * n_node + node).
        flags & F_EXHAUSTIVE: spec §12 — unsuitable only if NO assignment of the pod exists."""
        c = np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
        po = np.ascontiguousarray(pod_off, dtype=np.uint32)
        if cand_nodes is None:
            n_pair = (len(po) - 1) * self.n_node
            bits = np.zeros((n_pair + 7) // 8 + 8, dtype=np.uint8)
            self._check(self._lib.dra_unsuitable_batch(self._h, _ptr(c), len(c), _ptr(po), len(po) - 1, None, None, _ptr(bits), flags))
            return bits[: (n_pair + 7) // 8]
        cn = np.ascontiguousarray(cand_nodes, dtype=np.uint32)
        co = np.ascontiguousarray(cand_off, dtype=np.uint32)
        n_pair = int(co[-1])
        bits = np.zeros((n_pair + 7) // 8 + 8, dtype=np.uint8)
        self._check(self._lib.dra_unsuitable_batch(self._h, _ptr(c), len(c), _ptr(po), len(po) - 1,
                                                   _ptr(cn), _ptr(co), _ptr(bits), flags))
        return bits[: (n_pair + 7) // 8]

    def preempt(self, claims, pod_off, prio, run_claims, run_pod_off, run_prio, run_out, run_out_off=None,
                cand_nodes=None, cand_off=None, max_victims: int = 8, flags: int = 0):
        """Preemption (spec §14): for each pending pod, the lower-priority running pods to evict on each candidate node and
        the node to evict them on.  The running pods are the arrays dra_deallocate_batch takes (run_claims, run_out,
        run_out_off) split by run_pod_off, index order = start order.  cand_nodes/cand_off None = every node, ascending.
        Returns (pair_status, pair_victims, pod_node, pod_status, n_victims, victims); victims is [n_pod, max_victims]
        with 0xFFFFFFFF past the end of a row, n_victims the full count."""
        c = np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
        po = np.ascontiguousarray(pod_off, dtype=np.uint32)
        pr = np.ascontiguousarray(prio, dtype=np.int32)
        n_pod = len(po) - 1
        run = _running(run_claims, run_pod_off, run_prio, run_out, run_out_off)
        cn, co = _cands(cand_nodes, cand_off)
        n_pair = n_pod * self.n_node if co is None else int(co[-1])
        pair_status = np.zeros(max(n_pair, 1), dtype=np.uint8)
        pair_victims = np.zeros(max(n_pair, 1), dtype=np.uint32)
        pod_node = np.zeros(max(n_pod, 1), dtype=np.uint32)
        pod_status = np.zeros(max(n_pod, 1), dtype=np.uint8)
        n_victims = np.zeros(max(n_pod, 1), dtype=np.uint32)
        victims = np.zeros(max(n_pod * max_victims, 1), dtype=np.uint32)
        self._check(self._lib.dra_preempt_batch(self._h, _ptr(c), len(c), _ptr(po), _ptr(pr), n_pod, _ptr(cn), _ptr(co),
                                                C.byref(run), _ptr(pair_status), _ptr(pair_victims), _ptr(pod_node),
                                                _ptr(pod_status), _ptr(n_victims), _ptr(victims) if max_victims else None,
                                                max_victims, flags))
        return (pair_status[:n_pair], pair_victims[:n_pair], pod_node[:n_pod], pod_status[:n_pod], n_victims[:n_pod],
                victims[:n_pod * max_victims].reshape(n_pod, max_victims))

    def preempt_pdb(self, claims, pod_off, prio, run_claims, run_pod_off, run_prio, run_out, run_pdb, pdb_allowed,
                    run_out_off=None, cand_nodes=None, cand_off=None, max_victims: int = 8, flags: int = 0):
        """preempt() with disruption budgets (spec §14, "Disruption budgets"): run_pdb[r] the budget running pod r counts
        against (PDB_NONE for none; None: no array), pdb_allowed[b] each budget's disruptionsAllowed (None: no budgets).
        Returns preempt()'s six outputs, then pair_violations and pod_violations (uint32).  Raises ValueError when run_pdb
        is given and does not hold one entry per running pod (the library reads one per running pod)."""
        c = np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
        po = np.ascontiguousarray(pod_off, dtype=np.uint32)
        pr = np.ascontiguousarray(prio, dtype=np.int32)
        n_pod = len(po) - 1
        run = _running(run_claims, run_pod_off, run_prio, run_out, run_out_off)
        rp = None if run_pdb is None else np.ascontiguousarray(run_pdb, dtype=np.uint32)
        if rp is not None and len(rp) != run.n_pod:
            raise ValueError(f"run_pdb holds {len(rp)} entries for {run.n_pod} running pods")
        al = None if pdb_allowed is None else np.ascontiguousarray(pdb_allowed, dtype=np.int32)
        bud = DisruptionBudgets(None if rp is None or not len(rp) else rp.ctypes.data,
                                None if al is None or not len(al) else al.ctypes.data, 0 if al is None else len(al))
        cn, co = _cands(cand_nodes, cand_off)
        n_pair = n_pod * self.n_node if co is None else int(co[-1])
        pair_status = np.zeros(max(n_pair, 1), dtype=np.uint8)
        pair_victims = np.zeros(max(n_pair, 1), dtype=np.uint32)
        pair_viol = np.zeros(max(n_pair, 1), dtype=np.uint32)
        pod_node = np.zeros(max(n_pod, 1), dtype=np.uint32)
        pod_status = np.zeros(max(n_pod, 1), dtype=np.uint8)
        n_victims = np.zeros(max(n_pod, 1), dtype=np.uint32)
        pod_viol = np.zeros(max(n_pod, 1), dtype=np.uint32)
        victims = np.zeros(max(n_pod * max_victims, 1), dtype=np.uint32)
        self._check(self._lib.dra_preempt_pdb_batch(
            self._h, _ptr(c), len(c), _ptr(po), _ptr(pr), n_pod, _ptr(cn), _ptr(co), C.byref(run), C.byref(bud),
            _ptr(pair_status), _ptr(pair_victims), _ptr(pair_viol), _ptr(pod_node), _ptr(pod_status), _ptr(n_victims),
            _ptr(pod_viol), _ptr(victims) if max_victims else None, max_victims, flags))
        return (pair_status[:n_pair], pair_victims[:n_pair], pod_node[:n_pod], pod_status[:n_pod], n_victims[:n_pod],
                victims[:n_pod * max_victims].reshape(n_pod, max_victims), pair_viol[:n_pair], pod_viol[:n_pod])

    def preempt_place(self, claims, pod_off, prio, run_claims, run_pod_off, run_prio, run_out, run_out_off=None,
                      cand_nodes=None, cand_off=None, out_off=None, n_out=None, flags: int = 0):
        """Preempt and place (spec §15): pods in input order, each judged as preempt() judges it on the inventory the pods
        before it left (their placements held, their victims gone), then applied: its victims released, the pod allocated
        on the chosen node.  Running pods as preempt() takes them; candidates and out_off / n_out as place_pods().  The
        call releases the victims itself: do not deallocate them again.  Returns (out, pod_node, pod_status, evicted_by);
        evicted_by[r] = the pod that evicted running pod r, 0xFFFFFFFF when none.  flags: 0 or F_EXHAUSTIVE."""
        c = np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
        po = np.ascontiguousarray(pod_off, dtype=np.uint32)
        pr = np.ascontiguousarray(prio, dtype=np.int32)
        n_pod = len(po) - 1
        oo = None if out_off is None else np.ascontiguousarray(out_off, dtype=np.uint32)
        if n_out is None:
            n_out = _placed_n_out(c, oo)
        run = _running(run_claims, run_pod_off, run_prio, run_out, run_out_off)
        cn, co = _cands(cand_nodes, cand_off)
        out = np.zeros(max(n_out, 1), dtype=R.OUT_DTYPE)
        pod_node = np.zeros(max(n_pod, 1), dtype=np.uint32)
        pod_status = np.zeros(max(n_pod, 1), dtype=np.uint8)
        evicted_by = np.zeros(max(run.n_pod, 1), dtype=np.uint32)
        self._check(self._lib.dra_preempt_place_batch(self._h, _ptr(c), len(c), _ptr(po), _ptr(pr), n_pod, _ptr(cn), _ptr(co),
                                                      C.byref(run), _ptr(oo), _ptr(out), n_out, _ptr(pod_node),
                                                      _ptr(pod_status), _ptr(evicted_by), flags))
        return out[:n_out], pod_node[:n_pod], pod_status[:n_pod], evicted_by[:run.n_pod]

    def pod_capacity(self, claims, pod_off, cand_nodes=None, cand_off=None, max_copies: int = 64, exhaustive: bool = False,
                     want_stop: bool = True, want_totals: bool = True):
        """Pod capacity (spec §16): how many copies of each pod every candidate node still takes, counted as
        allocate_pods() would place them (at most max_copies, 1 .. 65535).  cand_nodes/cand_off None = every node, pair
        k = pod * n_node + node.  Pure.  Returns (pair_copies u16, pair_stop u8 or None, pod_total u64 or None, pod_nodes
        u32 or None); pair_stop: ST_OK max_copies reached, ST_POD the next copy does not fit, ST_SEARCH_LIMIT its search
        ran out of budget, ST_INVALID."""
        c = np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
        po = np.ascontiguousarray(pod_off, dtype=np.uint32)
        n_pod = len(po) - 1
        cn, co = _cands(cand_nodes, cand_off)
        n_pair = n_pod * self.n_node if co is None else int(co[-1])
        copies = np.zeros(max(n_pair, 1), dtype=np.uint16)
        stop = np.zeros(max(n_pair, 1), dtype=np.uint8) if want_stop else None
        total = np.zeros(max(n_pod, 1), dtype=np.uint64) if want_totals else None
        nodes = np.zeros(max(n_pod, 1), dtype=np.uint32) if want_totals else None
        self._check(self._lib.dra_pod_capacity_batch(self._h, _ptr(c), len(c), _ptr(po), n_pod, _ptr(cn), _ptr(co), max_copies,
                                                     _ptr(copies), _ptr(stop), _ptr(total), _ptr(nodes),
                                                     F_EXHAUSTIVE if exhaustive else 0))
        return (copies[:n_pair], None if stop is None else stop[:n_pair], None if total is None else total[:n_pod],
                None if nodes is None else nodes[:n_pod])

    def deallocate(self, claims, out, out_off=None):
        """Spec §9: release the OK records `out` of `claims` (slots counted as Allocate counts them).  A claim whose slot
        range leaves [0, len(out)) raises DraError(DRA_E_INVAL) before anything is launched: the inventory is unchanged."""
        c = np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
        o = np.ascontiguousarray(out, dtype=R.OUT_DTYPE)
        oo = None if out_off is None else np.ascontiguousarray(out_off, dtype=np.uint32)
        self._check(self._lib.dra_deallocate_batch(self._h, _ptr(c), len(c), _ptr(oo), _ptr(o), len(o)))

    # -- adjacent integer searches ------------------------------------------------------------------------
    def mps_limits(self, nbytes) -> tuple:
        b = np.ascontiguousarray(nbytes, dtype=np.int64)
        mib = np.zeros(len(b), dtype=np.int64); valid = np.zeros(len(b), dtype=np.uint8)
        self._check(self._lib.dra_mps_limits_batch(self._h, _ptr(b), len(b), _ptr(mib), _ptr(valid)))
        return mib, valid.astype(bool)

    def imex_offsets(self, used_lists, step: int = 128, limit: int = 2048) -> np.ndarray:
        off = np.zeros(len(used_lists) + 1, dtype=np.uint32)
        off[1:] = np.cumsum([len(u) for u in used_lists])
        used = np.ascontiguousarray(np.concatenate([np.asarray(u, dtype=np.int32) for u in used_lists]) if len(used_lists) and off[-1] else np.zeros(1, np.int32), dtype=np.int32)
        out = np.zeros(len(used_lists), dtype=np.int32)
        self._check(self._lib.dra_imex_offsets_batch(self._h, _ptr(used), _ptr(off), len(used_lists), step, limit, _ptr(out)))
        return out

    # -- multi-GPU ------------------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        rc = load().dra_comm_unique_id(C.cast(buf, C.c_void_p))
        if rc != OK:
            raise DraError(rc, (load().dra_last_error(None) or b"").decode())
        return bytes(buf)

    def comm_init(self, uid: bytes, rank: int, world: int):
        buf = (C.c_uint8 * 128).from_buffer_copy(uid)
        self._check(self._lib.dra_comm_init(self._h, C.cast(buf, C.c_void_p), rank, world))

    def peer_rendezvous(self) -> None:
        """Enqueue a device-side rendezvous of all ranks on this context's stream (dra_peer_rendezvous_device)."""
        self._check(self._lib.dra_peer_rendezvous_device(self._h))

    def gather_read(self, out_all: np.ndarray) -> np.ndarray:
        """D2H of the last gather's table into out_all (OUT_DTYPE, world * n_per_rank); synchronises."""
        self._check(self._lib.dra_gather_read(self._h, _ptr(out_all), len(out_all)))
        return out_all

    def peer_disable(self) -> None:
        self._check(self._lib.dra_peer_export(self._h, 0, None))

    def peer_export(self, n_per_rank: int) -> bytes:
        buf = (C.c_uint8 * 64)()
        self._check(self._lib.dra_peer_export(self._h, n_per_rank, C.cast(buf, C.c_void_p)))
        return bytes(buf)

    def comm_init_local(self, rank: int, world: int) -> None:
        """Rank / world of a context whose peers live in THIS process (no NCCL communicator)."""
        self._check(self._lib.dra_comm_init_local(self._h, rank, world))

    def peer_import_local(self, ctxs) -> None:
        """Map the gather buffers of the world contexts of this process (rank order)."""
        arr = (C.c_void_p * len(ctxs))(*[c._h for c in ctxs])
        self._check(self._lib.dra_peer_import_local(self._h, C.cast(arr, C.c_void_p)))

    def set_shard(self, node_lo: int, node_hi: int, take_stray: bool = False) -> None:
        self._check(self._lib.dra_set_shard(self._h, node_lo, node_hi, 1 if take_stray else 0))

    def set_shard_map(self, bounds, stray_rank: int = 0) -> None:
        """bounds: world + 1 node indices; this rank serves [bounds[rank], bounds[rank + 1])."""
        b = np.ascontiguousarray(bounds, dtype=np.uint32)
        self._check(self._lib.dra_set_shard_map(self._h, _ptr(b), stray_rank))

    def shard_export(self, n_out_max: int, cap_per_rank: int = 0, want_handle: bool = True) -> bytes:
        buf = (C.c_uint8 * 64)()
        self._check(self._lib.dra_shard_export(self._h, n_out_max, cap_per_rank, C.cast(buf, C.c_void_p) if want_handle else None))
        return bytes(buf)

    def allocate_global_device(self, d_claims: int, n_claim: int, d_out_off: int | None, n_out: int, flags: int = 0):
        """Sharded global batch: the SAME claim array on every rank (device pointer); enqueues, no synchronisation.
        The result table: gather_read()."""
        self._check(self._lib.dra_allocate_batch_global_device(self._h, _ptr(d_claims), n_claim, _ptr(d_out_off), n_out, flags))

    def set_shard_pairs(self, max_pairs: int) -> None:
        """Room for the sharded UnsuitableNodes bit exchange; world > 1: before shard_export, the same on every rank."""
        self._check(self._lib.dra_set_shard_pairs(self._h, max_pairs))

    def unsuitable_global_device(self, d_claims: int, n_claim: int, d_pod_off: int, n_pod: int, d_cand_nodes: int | None,
                                 d_cand_off: int | None, n_pair: int, d_bits: int, flags: int = 0) -> None:
        """Sharded UnsuitableNodes: the SAME pods and candidates on every rank (device pointers); every rank receives the
        whole bitmap, ceil(n_pair / 8) bytes at d_bits.  d_cand_nodes / d_cand_off None = dense form (n_pair = n_pod *
        n_node).  Enqueues, no synchronisation; errors found on the device surface at sync()."""
        self._check(self._lib.dra_unsuitable_batch_global_device(self._h, _ptr(d_claims), n_claim, _ptr(d_pod_off), n_pod,
                                                                 _ptr(d_cand_nodes), _ptr(d_cand_off), n_pair, _ptr(d_bits),
                                                                 flags))

    def allocate_pods_global_device(self, d_claims: int, n_claim: int, d_pod_off: int, n_pod: int, d_out_off: int | None,
                                    n_out: int, flags: int = 0) -> None:
        """Sharded pods Allocate (spec §12): the SAME pods on every rank (device pointers); a pod is placed by the rank that
        owns its first claim's node, and every rank receives the whole table (gather_read()).  flags: F_EXHAUSTIVE,
        F_FRESH_INVENTORY.  Enqueues, no synchronisation; errors found on the device surface at sync()."""
        self._check(self._lib.dra_allocate_pods_batch_global_device(self._h, _ptr(d_claims), n_claim, _ptr(d_pod_off), n_pod,
                                                                    _ptr(d_out_off), n_out, flags))

    def set_shard_place(self, max_pods: int) -> None:
        """Room for the sharded place-pods call's replicated pod states; world > 1: before shard_export, the same on every
        rank."""
        self._check(self._lib.dra_set_shard_place(self._h, max_pods))

    def place_pods_global_device(self, d_claims: int, n_claim: int, d_pod_off: int, n_pod: int, d_cand_nodes: int | None,
                                 d_cand_off: int | None, n_pair: int, d_out_off: int | None, n_out: int, d_pod_node: int,
                                 flags: int = 0) -> None:
        """Sharded place pods (spec §13): the SAME pods and candidates on every rank (device pointers); d_cand_nodes /
        d_cand_off None and n_pair 0 = dense form.  Each rank evaluates the visits to its own nodes; every rank receives the
        whole table (gather_read()) and the whole pod_node array, n_pod uint32 at d_pod_node.  flags: F_EXHAUSTIVE,
        F_FRESH_INVENTORY.  Enqueues, no synchronisation; errors found on the device surface at sync()."""
        self._check(self._lib.dra_place_pods_batch_global_device(self._h, _ptr(d_claims), n_claim, _ptr(d_pod_off), n_pod,
                                                                 _ptr(d_cand_nodes), _ptr(d_cand_off), n_pair, _ptr(d_out_off),
                                                                 n_out, _ptr(d_pod_node), flags))

    def set_shard_preempt(self, max_pods: int, max_pairs: int, max_victims: int) -> None:
        """Room for the sharded preemption call's partials; world > 1: before shard_export, the same on every rank."""
        self._check(self._lib.dra_set_shard_preempt(self._h, max_pods, max_pairs, max_victims))

    def preempt_global_device(self, d_claims: int, n_claim: int, d_pod_off: int, d_prio: int, n_pod: int,
                              d_cand_nodes: int | None, d_cand_off: int | None, n_pair: int, running: "RunningPods",
                              d_pair_status: int | None, d_pair_victims: int | None, d_pod_node: int, d_pod_status: int,
                              d_n_victims: int, d_victims: int | None, max_victims: int, flags: int = 0) -> None:
        """Sharded preemption (spec §14): the SAME pending pods, candidates and running pods on every rank (device
        pointers; `running` a RunningPods whose pointers are device-visible).  d_cand_nodes / d_cand_off None = dense form
        (n_pair = n_pod * n_node).  Every rank receives the whole outputs, laid out as preempt()'s; the pair outputs may be
        None.  Enqueues, no synchronisation; errors found on the device surface at sync()."""
        self._check(self._lib.dra_preempt_batch_global_device(
            self._h, _ptr(d_claims), n_claim, _ptr(d_pod_off), _ptr(d_prio), n_pod, _ptr(d_cand_nodes), _ptr(d_cand_off),
            n_pair, C.byref(running), _ptr(d_pair_status), _ptr(d_pair_victims), _ptr(d_pod_node), _ptr(d_pod_status),
            _ptr(d_n_victims), _ptr(d_victims), max_victims, flags))

    def preempt_pdb_global_device(self, d_claims: int, n_claim: int, d_pod_off: int, d_prio: int, n_pod: int,
                                  d_cand_nodes: int | None, d_cand_off: int | None, n_pair: int, running: "RunningPods",
                                  budgets: "DisruptionBudgets | None", d_pair_status: int | None, d_pair_victims: int | None,
                                  d_pair_violations: int | None, d_pod_node: int, d_pod_status: int, d_n_victims: int,
                                  d_pod_violations: int | None, d_victims: int | None, max_victims: int,
                                  flags: int = 0) -> None:
        """preempt_global_device() with disruption budgets, as preempt_pdb() answers them: `budgets` a DisruptionBudgets
        whose pointers are device-visible (None: none), the same on every rank; the violation outputs (uint32) may be
        None.  Enqueues, no synchronisation; errors found on the device surface at sync()."""
        self._check(self._lib.dra_preempt_pdb_batch_global_device(
            self._h, _ptr(d_claims), n_claim, _ptr(d_pod_off), _ptr(d_prio), n_pod, _ptr(d_cand_nodes), _ptr(d_cand_off),
            n_pair, C.byref(running), None if budgets is None else C.byref(budgets), _ptr(d_pair_status),
            _ptr(d_pair_victims), _ptr(d_pair_violations), _ptr(d_pod_node), _ptr(d_pod_status), _ptr(d_n_victims),
            _ptr(d_pod_violations), _ptr(d_victims), max_victims, flags))

    def set_shard_capacity(self, max_pairs: int) -> None:
        """Room for the sharded pod-capacity call's pair results; world > 1: before shard_export, the same on every rank."""
        self._check(self._lib.dra_set_shard_capacity(self._h, max_pairs))

    def pod_capacity_global_device(self, d_claims: int, n_claim: int, d_pod_off: int, n_pod: int, d_cand_nodes: int | None,
                                   d_cand_off: int | None, n_pair: int, max_copies: int, d_pair_copies: int | None,
                                   d_pair_stop: int | None = None, d_pod_total: int | None = None,
                                   d_pod_nodes: int | None = None, flags: int = 0) -> None:
        """Sharded pod capacity (spec §16): the SAME pods and candidates on every rank (device pointers); d_cand_nodes /
        d_cand_off None = dense form (n_pair = n_pod * n_node).  Each rank counts the pairs of its own nodes; every rank
        receives the whole outputs, laid out as pod_capacity()'s (u16 copies, u8 stops, u64 totals, u32 node counts); all
        but d_pair_copies may be None.  Enqueues, no synchronisation; errors found on the device surface at sync()."""
        self._check(self._lib.dra_pod_capacity_batch_global_device(
            self._h, _ptr(d_claims), n_claim, _ptr(d_pod_off), n_pod, _ptr(d_cand_nodes), _ptr(d_cand_off), n_pair,
            max_copies, _ptr(d_pair_copies), _ptr(d_pair_stop), _ptr(d_pod_total), _ptr(d_pod_nodes), flags))

    def set_shard_preempt_place(self, max_pods: int, max_pairs: int, max_run: int) -> None:
        """Room for the sharded preempt-and-place call (pending pods, judged pairs, running pods); world > 1: before
        shard_export, with the inventory loaded, the same on every rank."""
        self._check(self._lib.dra_set_shard_preempt_place(self._h, max_pods, max_pairs, max_run))

    def preempt_place_global_device(self, d_claims: int, n_claim: int, d_pod_off: int, d_prio: int, n_pod: int,
                                    d_cand_nodes: int | None, d_cand_off: int | None, n_pair: int, running: "RunningPods",
                                    d_out_off: int | None, n_out: int, d_pod_node: int, d_pod_status: int,
                                    d_evicted_by: int | None, flags: int = 0) -> None:
        """Sharded preempt and place (spec §15): the SAME pending pods, candidates and running pods on every rank (device
        pointers; `running` a RunningPods whose pointers are device-visible); d_cand_nodes / d_cand_off None and n_pair 0 =
        dense form.  Every rank receives the whole table (gather_read()) and the whole pod_node (n_pod uint32), pod_status
        (n_pod uint8) and evicted_by (one uint32 per running pod); each rank's own GPU range ends as preempt_place() leaves
        it.  flags: F_EXHAUSTIVE.  Enqueues, no synchronisation; errors found on the device surface at sync()."""
        self._check(self._lib.dra_preempt_place_batch_global_device(
            self._h, _ptr(d_claims), n_claim, _ptr(d_pod_off), _ptr(d_prio), n_pod, _ptr(d_cand_nodes), _ptr(d_cand_off),
            n_pair, C.byref(running), _ptr(d_out_off), n_out, _ptr(d_pod_node), _ptr(d_pod_status), _ptr(d_evicted_by),
            flags))

    def shard_sync_inventory_device(self) -> None:
        """Every rank's live inventory becomes the world's state (each GPU as its owning rank holds it), so get_inventory()
        returns the whole world and set_shard_map() may move ranges without losing allocations.  Every rank must call it;
        one process: enqueue it on every rank before get_inventory() / set_shard_map() on any.  Enqueues, no
        synchronisation; errors found on the device surface at sync()."""
        self._check(self._lib.dra_shard_sync_inventory_device(self._h))

    def deallocate_global_device(self, d_claims: int, n_claim: int, d_out_off: int | None, d_out: int, n_out: int) -> None:
        """Sharded Deallocate (spec §9): the SAME claims, out_off and OutRecs on every rank (device pointers or PinnedBuffer
        addresses; d_out may be the gathered table).  This rank applies the OK records on its own GPU range and writes no
        other GPU.  A slot range outside n_out fails the call at sync() with no inventory changed.  Needs no export or
        import and waits for no peer.  Enqueues, no synchronisation."""
        self._check(self._lib.dra_deallocate_batch_global_device(self._h, _ptr(d_claims), n_claim, _ptr(d_out_off), _ptr(d_out),
                                                                 n_out))

    def peer_import(self, handles) -> None:
        blob = b"".join(handles)
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        self._check(self._lib.dra_peer_import(self._h, C.cast(buf, C.c_void_p)))

    def calibrate(self) -> int:
        """Measure the single-launch / sort-path crossover on this device + inventory; returns the claim count."""
        v = _u32(0)
        self._check(self._lib.dra_calibrate(self._h, C.byref(v)))
        return int(v.value)

    # -- resident mode ----------------------------------------------------------------------------------
    def serve_start(self) -> None:
        self._check(self._lib.dra_serve_start(self._h))

    def serve_stop(self) -> None:
        self._check(self._lib.dra_serve_stop(self._h))

    def serve_batches(self) -> int:
        return int(self._lib.dra_serve_batches(self._h))

    # -- instrumentation ------------------------------------------------------------------------------
    def launch_count(self) -> int:
        return int(self._lib.dra_launch_count(self._h))

    def set_profiling(self, on: bool):
        self._check(self._lib.dra_set_profiling(self._h, 1 if on else 0))

    def debug_noop(self, grid: int, block: int, smem: int) -> None:
        self._check(self._lib.dra_debug_noop(self._h, grid, block, smem))

    def last_chain(self) -> set:
        """Names (KERNELS keys) of the kernels the last Allocate-family call enqueued."""
        k = _u32(0)
        self._check(self._lib.dra_debug_last_chain(self._h, C.byref(k), None))
        return {n for n, bit in KERNELS.items() if k.value & bit}

    def last_hist_tile(self) -> int:
        """Claims per histogram tile of the last Allocate-family call (0: it ran no histogram kernel)."""
        t = _u32(0)
        self._check(self._lib.dra_debug_last_chain(self._h, None, C.byref(t)))
        return int(t.value)

    def debug_timeline(self, n_cta: int) -> np.ndarray:
        buf = np.zeros(n_cta * 8, dtype=np.uint64)
        n = self._lib.dra_debug_timeline(self._h, _ptr(buf), len(buf))
        return buf[:n].reshape(-1, 8)

    def debug_serve_times(self):
        buf = np.zeros(4, dtype=np.uint64)
        return buf if self._lib.dra_debug_serve_times(self._h, _ptr(buf)) == 4 else None

    def debug_shard_times(self):
        buf = np.zeros(2, dtype=np.uint64)
        return buf if self._lib.dra_debug_shard_times(self._h, _ptr(buf)) == 2 else None

    def timings_us(self) -> dict:
        buf = (C.c_float * 5)()
        n = self._lib.dra_get_timings(self._h, C.cast(buf, C.c_void_p), 5)
        names = ["bucket_hist", "bucket_scan", "bucket_scatter", "pack", "all_gather"]
        return {names[i]: float(buf[i]) for i in range(n)}
