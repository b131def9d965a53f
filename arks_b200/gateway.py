"""Host-side mirror of the reference's plugin seams over libarksgw.so (the C ABI in include/arks_gateway.h).

The reference wires three interfaces into its ext_proc server (cmd/gateway/main.go:233-270):
  ratelimiter.RateLimterInterface  (CheckLimit / DoLimit)            pkg/gateway/ratelimiter/rate_limiter.go:21-28
  quota.QuotaService               (IncrUsage / SetUsage / GetUsage) pkg/gateway/quota/types.go:24-28
  qosconfig.ConfigProvider         (GetQosByToken / GetQuotaConfig / GetModelList)  pkg/gateway/qosconfig/provider.go:29-37
On the GPU they are one object, because config, limiter windows and quota usage live together in HBM and a
request is decided in one pass over its body. `Gateway` is that object; `handle_request_body` /
`handle_response_body` keep the names of the Go handlers they batch (pkg/gateway/handle_request.go:83,
pkg/gateway/handle_response.go:80).

There is no CPU fallback: if the shared library or a CUDA device is missing, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import abi
from .abi import (ArksRequestBatch, ArksRequestResult, ArksResponseBatch, ArksResponseResult, ArksTables,
                  RequestBatch, RequestResult, ResponseBatch, ResponseResult)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ARKS_LIB", os.path.join(_HERE, "libarksgw.so"))  # ARKS_LIB: A/B builds in experiments
_lib = None


class ArksError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"arks error {code}: {msg}")
        self.code = code


def lib():
    """Load libarksgw.so (built in-tree by __graft_entry__.build()). Raises if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(LIB_PATH)
        vp = C.c_void_p
        L.arks_abi_version.restype = C.c_int
        L.arks_create.argtypes = [C.c_int, C.c_uint32, C.c_uint64, C.POINTER(vp)]
        L.arks_destroy.argtypes = [vp]
        L.arks_last_error.restype = C.c_char_p
        L.arks_last_error.argtypes = [vp]
        L.arks_load_tables.argtypes = [vp, C.POINTER(ArksTables)]
        L.arks_load_bpe.argtypes = [vp, vp]
        L.arks_load_bpe_vocab.argtypes = [vp, C.c_uint32, vp, abi.u8p, abi.u32p, C.c_uint32]
        L.arks_bind_model_vocab.argtypes = [vp, C.c_char_p, C.c_uint32, C.c_uint32]
        L.arks_prepare_tables.argtypes = [vp, C.POINTER(ArksTables), C.POINTER(vp)]
        L.arks_commit_tables.argtypes = [vp, vp]
        L.arks_discard_prepared.argtypes = [vp, vp]
        L.arks_discard_prepared.restype = None
        cp, u32 = C.c_char_p, C.c_uint32
        L.arks_upsert_token.argtypes = [vp, cp, u32, cp, u32, cp, u32, C.POINTER(abi.ArksQosSpec), u32]
        L.arks_upsert_quota.argtypes = [vp, cp, u32, cp, u32, abi.u8p, abi.i64p, u32]
        L.arks_upsert_endpoint.argtypes = [vp, cp, u32, cp, u32, abi.i32p, u32]
        for f in (L.arks_delete_token, L.arks_delete_quota, L.arks_delete_endpoint):
            f.argtypes = [vp, cp, u32, cp, u32]
        L.arks_config_prepare.argtypes = [vp, C.POINTER(vp)]
        L.arks_find_quota.argtypes = [vp, cp, u32, cp, u32]
        L.arks_find_quota.restype = C.c_int32
        L.arks_find_qos.argtypes = [vp, cp, u32, cp, u32, cp, u32]
        L.arks_find_qos.restype = C.c_int32
        L.arks_set_precharge.argtypes = [vp, C.c_int]
        L.arks_set_stream_metering.argtypes = [vp, C.c_int]
        L.arks_table_generation.restype = C.c_uint32
        L.arks_table_generation.argtypes = [vp]
        L.arks_update_endpoint_weights.argtypes = [vp, C.c_uint32, C.c_uint32, abi.i32p]
        L.arks_submit_request_batch.argtypes = [vp, C.POINTER(ArksRequestBatch), C.POINTER(ArksRequestResult)]
        L.arks_submit_response_batch.argtypes = [vp, C.POINTER(ArksResponseBatch), C.POINTER(ArksResponseResult)]
        L.arks_stage_request_batch.argtypes = [vp, C.POINTER(ArksRequestBatch)]
        L.arks_run_request_batch.argtypes = [vp, C.c_int64]
        L.arks_fetch_request_result.argtypes = [vp, C.POINTER(ArksRequestResult)]
        L.arks_stage_response_batch.argtypes = [vp, C.POINTER(ArksResponseBatch)]
        L.arks_run_response_batch.argtypes = [vp, C.c_int64]
        L.arks_fetch_response_result.argtypes = [vp, C.POINTER(ArksResponseResult)]
        L.arks_submit_request_async.argtypes = [vp, C.POINTER(ArksRequestBatch)]
        L.arks_wait_request.argtypes = [vp, C.c_int, C.POINTER(ArksRequestResult)]
        L.arks_submit_response_async.argtypes = [vp, C.POINTER(ArksResponseBatch)]
        L.arks_wait_response.argtypes = [vp, C.c_int, C.POINTER(ArksResponseResult)]
        L.arks_select_slot.argtypes = [vp, C.c_int]
        L.arks_set_profiling.argtypes = [vp, C.c_int]
        L.arks_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float), C.c_int]
        L.arks_stream.restype = vp
        L.arks_stream.argtypes = [vp]
        L.arks_last_declined.restype = C.c_int64
        L.arks_last_declined.argtypes = [vp]
        L.arks_launch_count.restype = C.c_uint64
        L.arks_launch_count.argtypes = [vp]
        L.arks_last_staging_route.restype = C.c_int
        L.arks_last_staging_route.argtypes = [vp]
        L.arks_snapshot_quota.argtypes = [vp, abi.i64p]
        L.arks_set_quota_usage.argtypes = [vp, C.c_uint32, abi.i64p]
        L.arks_incr_quota_usage.argtypes = [vp, C.c_uint32, abi.i64p]
        L.arks_snapshot_rate.argtypes = [vp, C.c_int64, abi.i64p]
        L.arks_sync_quota_usage.argtypes = [vp, C.c_int, abi.u32p, abi.i64p, abi.u8p]
        L.arks_enable_metrics.argtypes = [vp, C.c_int]
        L.arks_snapshot_metrics.argtypes = [vp, abi.i64p]
        L.arks_enable_quota_sharing.argtypes = [vp, C.c_int]
        L.arks_take_quota_delta.argtypes = [vp, abi.i64p]
        L.arks_apply_quota_delta.argtypes = [vp, abi.i64p]
        L.arks_export_quota_delta_dev.argtypes = [vp, vp]
        L.arks_fold_quota_delta_dev.argtypes = [vp, vp, vp]
        L.arks_comm_unique_id.argtypes = [vp, vp]
        L.arks_comm_init.argtypes = [vp, C.c_int, C.c_int, vp, abi.u32p, C.c_uint32]
        L.arks_comm_set_shared.argtypes = [vp, abi.u32p, C.c_uint32]
        L.arks_fold_quota_allreduce.argtypes = [vp, C.c_int]
        L.arks_comm_destroy.argtypes = [vp]
        L.arks_comm_destroy.restype = None
        L.arks_extract_bearer.restype = C.c_size_t
        _lib = L
    return _lib


EXPORTED = [  # every symbol include/arks_gateway.h declares (checked by tests/test_abi.py)
    "arks_abi_version", "arks_create", "arks_destroy", "arks_last_error", "arks_load_tables", "arks_table_generation", "arks_load_bpe", "arks_set_precharge",
    "arks_set_stream_metering", "arks_load_bpe_vocab", "arks_bind_model_vocab",
    "arks_prepare_tables", "arks_commit_tables", "arks_discard_prepared", "arks_upsert_token", "arks_delete_token", "arks_upsert_quota",
    "arks_delete_quota", "arks_upsert_endpoint", "arks_delete_endpoint", "arks_config_prepare", "arks_find_quota", "arks_find_qos",
    "arks_update_endpoint_weights", "arks_extract_bearer", "arks_submit_request_batch",
    "arks_submit_response_batch", "arks_stage_request_batch", "arks_run_request_batch",
    "arks_fetch_request_result", "arks_stage_response_batch", "arks_run_response_batch",
    "arks_fetch_response_result", "arks_submit_request_async", "arks_wait_request", "arks_submit_response_async",
    "arks_wait_response", "arks_select_slot", "arks_set_profiling", "arks_last_kernel_ms", "arks_stream", "arks_launch_count", "arks_last_declined", "arks_last_staging_route", "arks_enable_metrics", "arks_snapshot_metrics", "arks_sync_quota_usage", "arks_alloc_pinned", "arks_free_pinned", "arks_snapshot_quota",
    "arks_set_quota_usage", "arks_incr_quota_usage", "arks_snapshot_rate", "arks_take_quota_delta",
    "arks_apply_quota_delta", "arks_quota_delta_dev", "arks_fold_quota_delta_dev", "arks_enable_quota_sharing",
    "arks_comm_unique_id", "arks_comm_init", "arks_comm_set_shared", "arks_fold_quota_allreduce", "arks_comm_destroy",
    "arks_export_quota_delta_dev",
]


class Gateway:
    """One per GPU. All mutable gateway state (rate windows, quota usage) lives in this object's HBM."""

    def __init__(self, device: int = 0, max_batch: int = 65536, max_batch_bytes: int = 96 << 20,
                 share_quota: bool = False):
        self._h = C.c_void_p()
        rc = lib().arks_create(device, max_batch, max_batch_bytes, C.byref(self._h))
        if not rc and share_quota:
            rc = lib().arks_enable_quota_sharing(self._h, 1)
        if rc:
            msg = lib().arks_last_error(self._h).decode() if self._h else "no CUDA device (there is no CPU fallback)"
            h, self._h = self._h, C.c_void_p()
            if h:
                lib().arks_destroy(h)
            raise ArksError(rc, msg)
        self.tables = None

    def close(self):
        if getattr(self, "_h", None):
            lib().arks_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc:
            raise ArksError(rc, lib().arks_last_error(self._h).decode())

    # ---- qosconfig.ConfigProvider: informer snapshot -> HBM tables
    def load_tables(self, tables):
        ts = tables.c_struct()
        self._ck(lib().arks_load_tables(self._h, C.byref(ts)))
        self.tables = tables

    def prepare_tables(self, tables):
        """config thread: build + upload the next generation off the data path -> opaque handle for commit_tables"""
        ts = tables.c_struct()
        h = C.c_void_p()
        self._ck(lib().arks_prepare_tables(self._h, C.byref(ts), C.byref(h)))
        return (h, tables)

    def commit_tables(self, prepared):
        """batch thread, between two submissions: stream-ordered swap, counters carried by key on the device, no host wait"""
        h, tables = prepared
        self._ck(lib().arks_commit_tables(self._h, h))
        if tables is not None:
            self.tables = tables

    def discard_prepared(self, prepared):
        lib().arks_discard_prepared(self._h, prepared[0])

    # ---- one informer event = one call (qosconfig/arks_impl.go:104-189); config_prepare() + commit_tables() publish them
    def upsert_token(self, namespace: str, name: str, token: str, qos):
        """qos: [(model, quota_name or "", [(rule, limit), ...]), ...]"""
        specs = (abi.ArksQosSpec * max(1, len(qos)))()
        keep = []
        for i, (model, quota, rls) in enumerate(qos):
            m, q = model.encode(), (quota or "").encode()
            rr = np.array([r for r, _ in rls], np.uint8)
            rv = np.array([v for _, v in rls], np.int64)
            keep += [m, q, rr, rv]
            specs[i] = abi.ArksQosSpec(m, len(m), q, len(q), len(rls), abi.ptr(rr, abi.u8p), abi.ptr(rv, abi.i64p))
        ns, nm, tk = namespace.encode(), name.encode(), token.encode()
        self._ck(lib().arks_upsert_token(self._h, ns, len(ns), nm, len(nm), tk, len(tk), specs, len(qos)))

    def upsert_quota(self, namespace: str, name: str, items):
        """items: [(quota_type, limit), ...]"""
        t = np.array([a for a, _ in items], np.uint8)
        v = np.array([b for _, b in items], np.int64)
        ns, nm = namespace.encode(), name.encode()
        self._ck(lib().arks_upsert_quota(self._h, ns, len(ns), nm, len(nm), abi.ptr(t, abi.u8p), abi.ptr(v, abi.i64p), len(items)))

    def upsert_endpoint(self, namespace: str, name: str, weights):
        w = np.ascontiguousarray(weights, np.int32)
        ns, nm = namespace.encode(), name.encode()
        self._ck(lib().arks_upsert_endpoint(self._h, ns, len(ns), nm, len(nm), abi.ptr(w, abi.i32p), len(w)))

    def delete_object(self, kind: str, namespace: str, name: str):
        f = {"token": lib().arks_delete_token, "quota": lib().arks_delete_quota, "endpoint": lib().arks_delete_endpoint}[kind]
        ns, nm = namespace.encode(), name.encode()
        self._ck(f(self._h, ns, len(ns), nm, len(nm)))

    def config_prepare(self):
        h = C.c_void_p()
        self._ck(lib().arks_config_prepare(self._h, C.byref(h)))
        return (h, None)

    def find_quota(self, namespace: str, name: str) -> int:
        ns, nm = namespace.encode(), name.encode()
        return int(lib().arks_find_quota(self._h, ns, len(ns), nm, len(nm)))

    def find_qos(self, namespace: str, user: str, model: str) -> int:
        ns, u, m = namespace.encode(), user.encode(), model.encode()
        return int(lib().arks_find_qos(self._h, ns, len(ns), u, len(u), m, len(m)))

    def load_bpe(self, tables):
        """switch the bpe_count columns on with a vocabulary (arks_b200.bpe.BpeTables), or off with None"""
        if tables is None:
            self._ck(lib().arks_load_bpe(self._h, None))
            return
        ts = tables.c_struct()
        self._ck(lib().arks_load_bpe(self._h, C.byref(ts)))

    def load_bpe_vocab(self, slot: int, tables):
        """load a vocabulary (arks_b200.bpe.BpeTables) into slot 0..bpe.MAX_VOCABS-1, or empty the slot with None. Slot 0 is
        load_bpe's; the others need it and are counted for the models bound to them (bind_model_vocab)"""
        if tables is None:
            self._ck(lib().arks_load_bpe_vocab(self._h, slot, None, None, None, 0))
            return
        ts = tables.c_struct()
        tb, to = tables.tok_bytes, tables.tok_off
        n_tok = 0 if to is None else len(to) - 1
        self._ck(lib().arks_load_bpe_vocab(self._h, slot, C.byref(ts), abi.ptr(tb, abi.u8p), abi.ptr(to, abi.u32p), n_tok))

    def bind_model_vocab(self, model: str, slot: int):
        """config thread: count the model's rows with the vocabulary in `slot` (0: remove the binding) from the next
        generation on (load_tables / commit_tables)"""
        m = model.encode()
        self._ck(lib().arks_bind_model_vocab(self._h, m, len(m), slot))

    def set_precharge(self, on: bool):
        """N4, opt-in: admitted requests charge their prompt's BPE count to tpm / tpd when their batch commits; responses that
        carry `precharged` reconcile (needs load_bpe; changes admit / deny against the reference)"""
        self._ck(lib().arks_set_precharge(self._h, int(bool(on))))

    def set_stream_metering(self, on: bool):
        """N5, opt-in: stream requests without stream_options.include_usage are decided instead of refused and billed by their
        BPE counts (result flags & abi.FLAG_METERED; the host must set abi.RESP_METERED on every chunk of such a stream).
        Needs load_bpe"""
        self._ck(lib().arks_set_stream_metering(self._h, int(bool(on))))

    @property
    def generation(self) -> int:
        """table generation the qos / token indices of request results refer to (carry it with the stream)"""
        return int(lib().arks_table_generation(self._h))

    def update_endpoint_weights(self, endpoint: int, weights):
        w = np.ascontiguousarray(weights, np.int32)
        self._ck(lib().arks_update_endpoint_weights(self._h, endpoint, len(w), abi.ptr(w, abi.i32p)))

    # ---- HandleRequestBody for a micro-batch of streams
    def handle_request_body(self, b: RequestBatch, out: RequestResult | None = None) -> RequestResult:
        r = out if out is not None else RequestResult.empty(b.n)
        bs, rs = b.c_struct(), r.c_struct()
        self._ck(lib().arks_submit_request_batch(self._h, C.byref(bs), C.byref(rs)))
        return r

    # ---- HandleResponseBody (status 200) for a micro-batch of chunks / complete bodies
    def handle_response_body(self, b: ResponseBatch, out: ResponseResult | None = None) -> ResponseResult:
        r = out if out is not None else ResponseResult.empty(b.n)
        bs, rs = b.c_struct(), r.c_struct()
        self._ck(lib().arks_submit_response_batch(self._h, C.byref(bs), C.byref(rs)))
        return r

    # ---- asynchronous form: one batch in flight per staging slot
    def submit_request_async(self, b: RequestBatch):
        bs = b.c_struct()
        self._ck(lib().arks_submit_request_async(self._h, C.byref(bs)))

    def wait_request(self, slot: int, out: RequestResult) -> RequestResult:
        rs = out.c_struct()
        self._ck(lib().arks_wait_request(self._h, slot, C.byref(rs)))
        return out

    def submit_response_async(self, b: ResponseBatch):
        bs = b.c_struct()
        self._ck(lib().arks_submit_response_async(self._h, C.byref(bs)))

    def wait_response(self, slot: int, out: ResponseResult) -> ResponseResult:
        rs = out.c_struct()
        self._ck(lib().arks_wait_response(self._h, slot, C.byref(rs)))
        return out

    # ---- split form (bench: kernel-only timing with inputs resident in HBM)
    def stage_request(self, b: RequestBatch):
        bs = b.c_struct()
        self._ck(lib().arks_stage_request_batch(self._h, C.byref(bs)))

    def run_request(self, now_unix: int):
        self._ck(lib().arks_run_request_batch(self._h, int(now_unix)))

    def fetch_request(self, n: int, out: RequestResult | None = None) -> RequestResult:
        r = out if out is not None else RequestResult.empty(n)
        rs = r.c_struct()
        self._ck(lib().arks_fetch_request_result(self._h, C.byref(rs)))
        return r

    def stage_response(self, b: ResponseBatch):
        bs = b.c_struct()
        self._ck(lib().arks_stage_response_batch(self._h, C.byref(bs)))

    def run_response(self, now_unix: int):
        self._ck(lib().arks_run_response_batch(self._h, int(now_unix)))

    def fetch_response(self, n: int, out: ResponseResult | None = None) -> ResponseResult:
        r = out if out is not None else ResponseResult.empty(n)
        rs = r.c_struct()
        self._ck(lib().arks_fetch_response_result(self._h, C.byref(rs)))
        return r

    def select_slot(self, slot: int):
        self._ck(lib().arks_select_slot(self._h, int(slot)))

    def set_profiling(self, on: bool):
        self._ck(lib().arks_set_profiling(self._h, int(bool(on))))

    def last_kernel_ms(self):
        """request batch: [scan stage, rank + admit, fast-path kernel alone or 0, BPE kernels or 0]; response batch: the
        same without the admit entry; both + [meter kernel] when it ran (N5)"""
        buf = (C.c_float * 5)()
        n = lib().arks_last_kernel_ms(self._h, buf, 5)
        if n < 0:
            self._ck(n)
        return [float(buf[k]) for k in range(n)]

    @property
    def stream_handle(self) -> int:
        return int(lib().arks_stream(self._h) or 0)

    @property
    def last_declined(self) -> int:
        """rows of the last batch the fast path left to the exact engine (-1: the batch took the fused kernels)"""
        return int(lib().arks_last_declined(self._h))

    @property
    def launch_count(self) -> int:
        return int(lib().arks_launch_count(self._h))

    @property
    def last_staging_route(self) -> int:
        """where the last staged batch's bodies went: 0 the metadata upload (<= 16 KiB), 1 behind the metadata on the compute
        stream (<= 256 KiB), 2 the slot's bodies buffer; -1 nothing staged (empty or refused batch)"""
        return int(lib().arks_last_staging_route(self._h))

    # ---- quota.QuotaService surface + A14 snapshot
    def snapshot_quota(self) -> np.ndarray:
        out = np.zeros((self.tables.n_quotas, 3), np.int64)
        self._ck(lib().arks_snapshot_quota(self._h, abi.ptr(out, abi.i64p)))
        return out

    def sync_quota_usage(self, status_present: np.ndarray, status_used: np.ndarray, restore: bool = False) -> np.ndarray:
        """syncQuotaUsage over all ArksQuotas (arks_impl.go:217-300). status_present [n_quotas] uint32 bit masks and
        status_used [n_quotas, 3] int64 are updated in place (the CR status to write back); returns action[n_quotas]:
        bit0 update the CR, bit1 the store was outdated (reference: zeroed; restore=True: raised to the CR value)."""
        n = self.tables.n_quotas
        assert status_present.dtype == np.uint32 and status_used.dtype == np.int64 and status_used.shape == (n, 3)
        action = np.zeros(n, np.uint8)
        self._ck(lib().arks_sync_quota_usage(self._h, 1 if restore else 0, abi.ptr(status_present, abi.u32p),
                                             abi.ptr(status_used, abi.i64p), abi.ptr(action, abi.u8p)))
        return action

    def enable_metrics(self, on: bool = True):
        """accumulate the gateway's Prometheus series on the device (N3); off by default"""
        self._ck(lib().arks_enable_metrics(self._h, 1 if on else 0))

    def snapshot_metrics(self) -> np.ndarray:
        """[n_qos, METRIC_COLS] int64, layout abi.METRIC_*"""
        out = np.zeros((self.tables.n_qos, abi.METRIC_COLS), np.int64)
        self._ck(lib().arks_snapshot_metrics(self._h, abi.ptr(out, abi.i64p)))
        return out

    def snapshot_rate(self, now_unix: int) -> np.ndarray:
        out = np.zeros((self.tables.n_qos, 4), np.int64)
        self._ck(lib().arks_snapshot_rate(self._h, int(now_unix), abi.ptr(out, abi.i64p)))
        return out

    def set_quota_usage(self, quota: int, usage):
        u = np.ascontiguousarray(usage, np.int64)
        self._ck(lib().arks_set_quota_usage(self._h, quota, abi.ptr(u, abi.i64p)))

    def incr_quota_usage(self, quota: int, delta):
        u = np.ascontiguousarray(delta, np.int64)
        self._ck(lib().arks_incr_quota_usage(self._h, quota, abi.ptr(u, abi.i64p)))

    # ---- quotas shared across GPUs: delta exchange (sharding.QuotaDeltaExchange drives these)
    def take_quota_delta(self) -> np.ndarray:
        out = np.zeros((self.tables.n_quotas, 3), np.int64)
        self._ck(lib().arks_take_quota_delta(self._h, abi.ptr(out, abi.i64p)))
        return out

    def apply_quota_delta(self, remote):
        u = np.ascontiguousarray(remote, np.int64)
        self._ck(lib().arks_apply_quota_delta(self._h, abi.ptr(u, abi.i64p)))

    def export_quota_delta_dev(self, dst_ptr: int):
        self._ck(lib().arks_export_quota_delta_dev(self._h, C.c_void_p(dst_ptr)))

    def fold_quota_delta_dev(self, reduced_ptr: int, own_ptr: int = 0):
        """quota += reduced - own, delta -= own; own defaults to the library's copy of the last export"""
        self._ck(lib().arks_fold_quota_delta_dev(self._h, C.c_void_p(reduced_ptr), C.c_void_p(own_ptr) if own_ptr else None))

    # ---- the fold done by the library over NCCL (arks_comm_*): what a Go / C++ host calls; no torch on this path
    def comm_unique_id(self) -> bytes:
        buf = C.create_string_buffer(128)
        self._ck(lib().arks_comm_unique_id(self._h, buf))
        return buf.raw

    def comm_init(self, rank: int, world: int, unique_id: bytes, shared_local_idx=None):
        idx = None if shared_local_idx is None else np.ascontiguousarray(shared_local_idx, np.uint32)
        self._ck(lib().arks_comm_init(self._h, rank, world, unique_id, abi.ptr(idx, abi.u32p), 0 if idx is None else len(idx)))

    def comm_set_shared(self, shared_local_idx=None):
        idx = None if shared_local_idx is None else np.ascontiguousarray(shared_local_idx, np.uint32)
        self._ck(lib().arks_comm_set_shared(self._h, abi.ptr(idx, abi.u32p), 0 if idx is None else len(idx)))

    def fold_quota_allreduce(self, wait: bool = True):
        self._ck(lib().arks_fold_quota_allreduce(self._h, int(wait)))

    # ---- reply shaping helpers (what the Go host puts on the wire; handle_request.go:208-247, util.go:40-77)
    def request_headers(self, r: RequestResult, i: int) -> dict:
        """The three routing headers of an admitted request: model, namespace, username."""
        t = self.tables
        return {"model": t.qos_model_name[int(r.qos[i])], "namespace": t.token_namespace[int(r.token[i])],
                "username": t.token_user[int(r.token[i])]}


def extract_bearer(headers) -> bytes:
    """HandleRequestHeaders bearer extraction (handle_request.go:38-46) through the C ABI. headers: [(key, value)]."""
    n = len(headers)
    keys = [k if isinstance(k, bytes) else k.encode() for k, _ in headers]
    vals = [v if isinstance(v, bytes) else v.encode() for _, v in headers]
    kbuf = [C.create_string_buffer(k, max(len(k), 1)) for k in keys]
    vbuf = [C.create_string_buffer(v, max(len(v), 1)) for v in vals]
    KA = (C.c_void_p * max(n, 1))(*[C.addressof(b) for b in kbuf])
    VA = (C.c_void_p * max(n, 1))(*[C.addressof(b) for b in vbuf])
    KL = (C.c_size_t * max(n, 1))(*[len(k) for k in keys])
    VL = (C.c_size_t * max(n, 1))(*[len(v) for v in vals])
    tok = C.c_void_p()
    ln = lib().arks_extract_bearer(KA, KL, VA, VL, C.c_size_t(n), C.byref(tok))
    if not ln:
        return b""
    return C.string_at(tok.value, ln)
