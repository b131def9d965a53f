"""Config plane, host half (SURVEY.md section 8f N2): Kubernetes watch events for ArksToken / ArksQuota / ArksEndpoint ->
object-level upserts of the library -> one published table generation per burst of events; and the 10-second quota
status loop in the other direction.

Mirror of the reference's ArksProvider (pkg/gateway/qosconfig/arks_impl.go):
  * :104-189  controller-runtime informers on the three kinds; the event filter lets through creations, deletions and
              updates whose SPEC changed (GenerationChangedPredicate) -- status-only updates, which the provider itself
              writes every 10 s, never reach it. Readers see the informer cache, i.e. the latest object.
  * :217-300  syncQuotaUsage: list every ArksQuota, compare status.quotaStatus with the counters, raise the CR where the
              counters are ahead, (buggy) zero the counters where the CR is ahead; `restore=True` is the intended
              behaviour on start (the counters are raised to the CR).
Here the "cache" is the library's ConfigStore (arks_upsert_* / arks_delete_*), the snapshot the request path reads is a
table generation (arks_config_prepare + arks_commit_tables: built off the data path, swapped between two batches), and the
counters are the quota rows in HBM (arks_sync_quota_usage does the comparison for all quotas in one kernel).

The transport (client-go, an HTTP watch) is the embedder's: events arrive as the dicts of the Kubernetes watch wire format,
{"type": "ADDED" | "MODIFIED" | "DELETED" | "BOOKMARK" | "ERROR", "object": {...}}, lists as the `items` of a List call.
`gateway` is an arks_b200.gateway.Gateway (or anything with its config-plane methods); `publish(names)` is how the pending
upserts become the generation the batch thread reads (default: gateway.config_prepare + gateway.commit_tables; with the
compiled host it is arks_b200.cpphost.Batcher.apply_config, which builds on the calling thread and swaps between two cycles).
"""
from __future__ import annotations

import datetime
import queue
import sys
import threading
import time

import numpy as np

from . import abi
from .tables import Tables, endpoint_backends, endpoint_pricing

KINDS = {"ArksToken": "token", "ArksQuota": "quota", "ArksEndpoint": "endpoint"}
QUOTA_TYPE_NAMES = sorted(abi.QUOTA_TYPES, key=abi.QUOTA_TYPES.get)


def object_key(obj) -> tuple[str, str]:
    md = obj["metadata"]
    return md.get("namespace", "default"), md["name"]


def token_qos(obj):
    """ArksToken.spec.qos -> [(model, quota name or "", [(rule, limit), ...]), ...] (api/v1/arkstoken_types.go)"""
    return [(q["arksEndpoint"]["name"], (q.get("quota") or {}).get("name", "") or "",
             [(abi.RULES[r["type"]], int(r["value"])) for r in q.get("rateLimits") or []])
            for q in obj["spec"].get("qos") or []]


def quota_items(obj):
    return [(abi.QUOTA_TYPES[i["type"]], int(i["value"])) for i in obj["spec"].get("quotas") or []]


def _spec_of(kind, obj, ready_backends):
    """what the request path reads of an object: two events with the same value publish nothing"""
    if kind == "token":
        return (obj["spec"]["token"], token_qos(obj))
    if kind == "quota":
        return quota_items(obj)
    return endpoint_backends(obj, ready_backends) + (endpoint_pricing(obj),)


class ArksProvider:
    def __init__(self, gateway, publish=None, ready_backends=None, clock=None):
        self.g = gateway
        self._publish = publish or (lambda names: gateway.commit_tables((gateway.config_prepare()[0], names)))
        self.ready_backends = ready_backends  # {(namespace, endpoint): [services]}: what the ArksEndpoint controller discovered
        self._clock = clock or (lambda: datetime.datetime.now(datetime.timezone.utc))
        self._mu = threading.Lock()  # events, flushes and the status loop may come from different threads
        self.objects = {"token": {}, "quota": {}, "endpoint": {}}  # key -> latest object (the informer cache, host copy)
        self._spec = {"token": {}, "quota": {}, "endpoint": {}}   # key -> what was last pushed to the library
        self.dirty = False
        self.published = 0   # generations this provider published
        self.ignored = 0     # events that changed nothing the request path reads (status updates, bookmarks, resyncs)
        self.rejected = []   # (kind, key, error): objects the library or the conversion refused; the previous version stays

    # ---- watch events ----------------------------------------------------------------------------------------------
    def apply(self, event) -> bool:
        """one watch event; True when it changed the pending configuration (flush() will publish a generation)"""
        ty = event.get("type")
        if ty in ("BOOKMARK", "ERROR") or ty is None:
            self.ignored += 1
            return False
        obj = event["object"]
        kind = KINDS.get(obj.get("kind", ""))
        if kind is None:
            self.ignored += 1
            return False
        with self._mu:
            return self._delete(kind, obj) if ty == "DELETED" else self._upsert(kind, obj)

    def replace(self, kind_name: str, items) -> int:
        """the result of a List call (initial sync, or a relist after a watch expired): objects that are no longer listed are
        deleted, the others upserted; returns how many changed anything"""
        kind = KINDS[kind_name]
        n = 0
        with self._mu:
            listed = {object_key(o) for o in items}
            for k in [k for k in self.objects[kind] if k not in listed]:
                n += self._delete(kind, self.objects[kind][k])
            for o in items:
                n += self._upsert(kind, o)
        return n

    def _upsert(self, kind, obj) -> bool:
        k = object_key(obj)
        try:
            spec = _spec_of(kind, obj, self.ready_backends)
        except (KeyError, TypeError, ValueError) as e:  # a rule / quota type this gateway does not know, a missing field
            self._reject(kind, k, e)
            return False
        if self._spec[kind].get(k) == spec:
            self.objects[kind][k] = obj  # status and metadata stay current even when the spec did not move
            self.ignored += 1
            return False
        try:
            if kind == "token":
                self.g.upsert_token(k[0], k[1], spec[0], spec[1])
            elif kind == "quota":
                self.g.upsert_quota(k[0], k[1], spec)
            else:
                self.g.upsert_endpoint(k[0], k[1], spec[1])
                if spec[2] != self._price_of(k):
                    self.g.set_endpoint_price(k[0], k[1], *spec[2])
        except Exception as e:  # the library keeps the previous version of the object
            self._reject(kind, k, e)
            return False
        self.objects[kind][k] = obj
        self._spec[kind][k] = spec
        self.dirty = True
        return True

    def _price_of(self, k):
        """the price last pushed for endpoint k ((0, 0): none; only priced endpoints ever reach set_endpoint_price)"""
        spec = self._spec["endpoint"].get(k)
        return spec[2] if spec else (0, 0)

    def _reject(self, kind, k, e):
        self.rejected.append((kind, k, repr(e)))
        del self.rejected[:-256]  # a diagnostic, not a log: an object that is re-sent broken for days must not grow the process

    def _delete(self, kind, obj) -> bool:
        k = object_key(obj)
        self.objects[kind].pop(k, None)
        if kind == "endpoint" and self._price_of(k) != (0, 0):
            self.g.set_endpoint_price(k[0], k[1], 0, 0)
        if self._spec[kind].pop(k, None) is None:
            self.ignored += 1
            return False
        self.g.delete_object(kind, k[0], k[1])
        self.dirty = True
        return True

    def no_publish(self):
        """context manager: no generation is published while it is held (for readers of the CURRENT generation's rows that
        are not on the batch thread, e.g. a metrics scrape: the library's snapshot calls must not meet a table swap)"""
        return self._mu

    # ---- publishing ------------------------------------------------------------------------------------------------
    def tables(self) -> Tables:
        """the host-side names of the pending configuration, in the library's order ((namespace, name) per kind)"""
        srt = lambda d, live: [d[k] for k in sorted(live)]
        return Tables(srt(self.objects["token"], self._spec["token"]), srt(self.objects["quota"], self._spec["quota"]),
                      srt(self.objects["endpoint"], self._spec["endpoint"]), self.ready_backends)

    def flush(self) -> bool:
        """publish what accumulated since the last flush as ONE generation (a burst of events costs one swap); the build
        runs here, on the caller's (config) thread, the swap between two batches"""
        with self._mu:
            if not self.dirty:
                return False
            self._publish(self.tables())  # the names travel with the swap (gateway.tables / the host's reply shaping)
            self.dirty = False
        self.published += 1
        return True

    # ---- quota status loop (arks_impl.go:217-300) --------------------------------------------------------------------
    def sync_quota_status(self, restore: bool = False):
        """one pass of syncQuotaUsage over the published generation. Returns the status updates to send
        (`client.Status().Update`): [{"namespace", "name", "status": {"quotaStatus": [...]}}] for every ArksQuota whose status
        changed; the cached objects carry the new status too. restore=True on start: counters behind the CR are raised to it
        (the reference calls SetUsage with Request == 0 there, which zeroes them)."""
        with self._mu:
            t = self.g.tables
            n = t.n_quotas
            present = np.zeros(n, np.uint32)
            used = np.zeros((n, len(QUOTA_TYPE_NAMES)), np.int64)  # the token columns and the cost column
            objs = []
            for q in range(n):
                k = (t.strings[t.quota_ns_str[q]].decode(), t.strings[t.quota_name_str[q]].decode())
                o = self.objects["quota"].get(k)
                objs.append(o)
                seen = set()
                for s in ((o or {}).get("status") or {}).get("quotaStatus") or []:
                    ty = abi.QUOTA_TYPES.get(s.get("type"))
                    if ty is None or ty in seen:  # the reference stops at the first entry of a type
                        continue
                    seen.add(ty)
                    present[q] |= 1 << ty
                    used[q, ty] = int(s.get("used", 0))
            before_present, before_used = present.copy(), used.copy()
            action = self.g.sync_quota_usage(present, used, restore=restore)
            now = self._clock().strftime("%Y-%m-%dT%H:%M:%SZ")  # metav1.Time marshals as RFC 3339, seconds
            out = []
            for q in np.flatnonzero(action & 1):
                o = objs[q]
                if o is None:
                    continue
                status = [dict(s) for s in (o.get("status") or {}).get("quotaStatus") or []]
                seen = set()
                for s in status:
                    ty = abi.QUOTA_TYPES.get(s.get("type"))
                    if ty is None or ty in seen:
                        continue
                    seen.add(ty)
                    if used[q, ty] != before_used[q, ty]:
                        s["used"] = int(used[q, ty])
                        s["lastUpdateTime"] = now
                for ty, _ in quota_items(o):  # new entries in the order of spec.quotas
                    if ty not in seen and present[q] >> ty & 1 and not before_present[q] >> ty & 1:
                        seen.add(ty)
                        status.append({"type": QUOTA_TYPE_NAMES[ty], "used": int(used[q, ty]), "lastUpdateTime": now})
                o.setdefault("status", {})["quotaStatus"] = status
                ns, name = object_key(o)
                out.append({"namespace": ns, "name": name, "status": {"quotaStatus": status}})
            return out


class ProviderLoop:
    """What ArksProvider.Start leaves running (arks_impl.go:104-189): the event handler and the 10-second status ticker, as
    one loop on one config thread. Events are coalesced: a generation is published once no event has arrived for `debounce_s`
    (or `max_delay_s` after the first unpublished one, so a steady trickle cannot starve it). `write_status(updates)` sends
    the ArksQuota status updates (client.Status().Update); the first status pass runs in restore mode when
    `restore_on_start` is set."""

    def __init__(self, provider: ArksProvider, write_status=None, debounce_s=0.05, max_delay_s=1.0, sync_every_s=10.0,
                 restore_on_start=True):
        self.p, self.write_status = provider, write_status
        self.debounce_s, self.max_delay_s, self.sync_every_s = debounce_s, max_delay_s, sync_every_s
        self.restore_next = restore_on_start
        self.events: "queue.SimpleQueue" = queue.SimpleQueue()
        self.first_dirty = self.last_event = None
        self.next_sync = None
        self.stop = threading.Event()
        self.errors = []  # what run() survived

    def offer(self, event):
        """any thread (the watch connections)"""
        self.events.put(event)

    def step(self, now: float) -> float:
        """everything that is due at monotonic time `now`; returns when to come back at the latest"""
        while True:
            try:
                e = self.events.get_nowait()
            except queue.Empty:
                break
            if self.p.apply(e):
                self.last_event = now
                if self.first_dirty is None:
                    self.first_dirty = now
        if self.first_dirty is not None and (now - self.last_event >= self.debounce_s or now - self.first_dirty >= self.max_delay_s):
            self.p.flush()
            self.first_dirty = self.last_event = None
        if self.next_sync is None:
            self.next_sync = now + self.sync_every_s  # the ticker's first tick comes one period after the cache synced
        if now >= self.next_sync and self.p.g.tables is not None:
            updates = self.p.sync_quota_status(restore=self.restore_next)
            self.restore_next = False
            if updates and self.write_status:
                self.write_status(updates)
            self.next_sync = now + self.sync_every_s
        wake = self.next_sync
        if self.first_dirty is not None:
            wake = min(wake, self.last_event + self.debounce_s, self.first_dirty + self.max_delay_s)
        return wake

    def run(self):
        """until stop is set; 1 ms granularity while events are pending, asleep otherwise"""
        while not self.stop.is_set():
            now = time.monotonic()
            try:
                wake = self.step(now)
            except Exception as e:  # a refused generation or a failed status pass must not end the loop: retried in a second
                self.errors.append(repr(e))
                del self.errors[:-256]
                print(f"arks provider: {e!r}", file=sys.stderr)
                wake = now + 1.0
            self.stop.wait(max(0.001, min(wake - time.monotonic(), 0.05)))
