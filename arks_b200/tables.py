"""Config plane: ArksToken / ArksQuota / ArksEndpoint objects -> the flat `arks_tables` snapshot.

Host-side mirror of what the reference's ArksProvider keeps in its controller-runtime informer cache
(pkg/gateway/qosconfig/arks_impl.go:104-189, 303-397): objects are accepted in the CRD shape
(`metadata.name/namespace`, `spec.*`, exactly the YAML of examples/quickstart/quickstart.yaml:56-110) and
flattened once per config change, so the per-request path never touches object graphs.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from .abi import QUOTA_MISSING, QUOTA_NONE, QUOTA_TYPES, RULES, ArksTables, i32p, i64p, ptr, u8p, u32p


class Tables:
    """Flat snapshot + the python-side name lists needed to emit the model/namespace/username headers."""

    def __init__(self, tokens, quotas, endpoints, ready_backends=None):
        """tokens/quotas/endpoints: lists of CRD-shaped dicts.

        ready_backends: {(namespace, endpoint_name): [service names]} — ready ArksApplication services the
        ArksEndpoint controller would append at defaultWeight
        (internal/controller/arksendpoint_controller.go:293-347); static routeConfigs come first and shadow
        equally-named discovered services.
        """
        strs: list[bytes] = []
        index: dict[bytes, int] = {}

        def s(x) -> int:
            b = x if isinstance(x, bytes) else str(x).encode()
            i = index.get(b)
            if i is None:
                i = len(strs)
                index[b] = i
                strs.append(b)
            return i

        quota_index: dict[tuple[str, str], int] = {}
        q_ns, q_name, q_off, qi_type, qi_val = [], [], [0], [], []
        for q in quotas:
            md = q["metadata"]
            ns = md.get("namespace", "default")
            quota_index.setdefault((ns, md["name"]), len(q_ns))
            q_ns.append(s(ns))
            q_name.append(s(md["name"]))
            for it in q["spec"]["quotas"]:
                qi_type.append(QUOTA_TYPES[it["type"]])
                qi_val.append(int(it["value"]))
            q_off.append(len(qi_type))

        t_tok, t_ns, t_name, t_off = [], [], [], [0]
        qos_model, qos_quota, qos_rl_off, rl_rule, rl_val = [], [], [0], [], []
        self.token_namespace: list[str] = []
        self.token_user: list[str] = []
        self.qos_model_name: list[str] = []
        self.token_string: list[str] = []
        # what the 429 / 500 bodies name (ratelimiter/types.go:98-104, quota/types.go:41-55): per qos entry the rule names of
        # its rateLimits in order, its quota's name and the item types of that ArksQuota in order
        self.qos_rule_names: list[list[str]] = []
        self.qos_quota_name: list[str] = []
        self.qos_quota_item_types: list[list[str]] = []
        quota_items = {k: [it["type"] for it in quotas[v]["spec"]["quotas"]] for k, v in quota_index.items()}
        for t in tokens:
            md = t["metadata"]
            ns = md.get("namespace", "default")
            t_tok.append(s(t["spec"]["token"]))
            t_ns.append(s(ns))
            t_name.append(s(md["name"]))
            self.token_namespace.append(ns)
            self.token_user.append(md["name"])
            self.token_string.append(t["spec"]["token"])
            for qos in t["spec"].get("qos") or []:
                model = qos["arksEndpoint"]["name"]
                qos_model.append(s(model))
                self.qos_model_name.append(model)
                qname = (qos.get("quota") or {}).get("name", "")
                self.qos_rule_names.append([rl["type"] for rl in qos.get("rateLimits") or []])
                self.qos_quota_name.append(qname)
                self.qos_quota_item_types.append(quota_items.get((ns, qname), []))
                if qname == "":
                    qos_quota.append(QUOTA_NONE)
                else:
                    qos_quota.append(quota_index.get((ns, qname), QUOTA_MISSING))
                for rl in qos.get("rateLimits") or []:
                    rl_rule.append(RULES[rl["type"]])
                    rl_val.append(int(rl["value"]))
                qos_rl_off.append(len(rl_rule))
            t_off.append(len(qos_model))

        e_ns, e_name, e_off, b_w = [], [], [0], []
        self.endpoint_backends: list[list[str]] = []
        # (namespace, name) -> (prompt, completion) price per token of the priced endpoints (spec.pricing, `cost` quota items);
        # Gateway.load_tables / prepare_tables hand them to the library. The first object wins on duplicates, as in the lookup
        self.endpoint_price: dict[tuple[str, str], tuple[int, int]] = {}
        for e in endpoints:
            md = e["metadata"]
            ns = md.get("namespace", "default")
            price = endpoint_pricing(e)
            if price != (0, 0):
                self.endpoint_price.setdefault((ns, md["name"]), price)
            e_ns.append(s(ns))
            e_name.append(s(md["name"]))
            names, weights = endpoint_backends(e, ready_backends)
            b_w += weights
            self.endpoint_backends.append(names)
            e_off.append(len(b_w))

        self.strings = strs
        a = np.ascontiguousarray
        self.str_off = np.zeros(len(strs) + 1, np.uint32)
        if strs:
            self.str_off[1:] = np.cumsum([len(x) for x in strs])
        self.str_bytes = np.frombuffer(b"".join(strs) + b"\0", dtype=np.uint8).copy()
        self.tok_token_str = a(t_tok, np.uint32)
        self.tok_ns_str = a(t_ns, np.uint32)
        self.tok_name_str = a(t_name, np.uint32)
        self.tok_qos_off = a(t_off, np.uint32)
        self.qos_model_str = a(qos_model, np.uint32)
        self.qos_quota = a(qos_quota, np.int32)
        self.qos_rl_off = a(qos_rl_off, np.uint32)
        self.rl_rule = a(rl_rule, np.uint8)
        self.rl_value = a(rl_val, np.int64)
        self.quota_ns_str = a(q_ns, np.uint32)
        self.quota_name_str = a(q_name, np.uint32)
        self.quota_item_off = a(q_off, np.uint32)
        self.qitem_type = a(qi_type, np.uint8)
        self.qitem_value = a(qi_val, np.int64)
        self.ep_ns_str = a(e_ns, np.uint32)
        self.ep_name_str = a(e_name, np.uint32)
        self.ep_backend_off = a(e_off, np.uint32)
        self.backend_weight = a(b_w, np.int32)
        self.n_tokens, self.n_qos, self.n_quotas, self.n_endpoints = len(t_tok), len(qos_model), len(q_ns), len(e_ns)
        self.qos_token = np.repeat(np.arange(self.n_tokens, dtype=np.int32), np.diff(self.tok_qos_off).astype(np.int64))

    def names_blob(self) -> bytes:
        """the name tables of host/cpp (arks_host::ParseNameTables): one line per ArksToken / qos entry"""
        lines = ["T\t%s\t%s" % (ns, u) for ns, u in zip(self.token_namespace, self.token_user)]
        for q in range(self.n_qos):
            lines.append("Q\t%d\t%s\t%s\t%s\t%s" % (int(self.qos_token[q]), self.qos_model_name[q], self.qos_quota_name[q],
                                                    ",".join(self.qos_rule_names[q]), ",".join(self.qos_quota_item_types[q])))
        return "\n".join(lines).encode()

    def c_struct(self) -> ArksTables:
        return ArksTables(
            ptr(self.str_bytes, u8p), ptr(self.str_off, u32p), len(self.strings),
            self.n_tokens, ptr(self.tok_token_str, u32p), ptr(self.tok_ns_str, u32p), ptr(self.tok_name_str, u32p),
            ptr(self.tok_qos_off, u32p),
            self.n_qos, ptr(self.qos_model_str, u32p), ptr(self.qos_quota, i32p), ptr(self.qos_rl_off, u32p),
            len(self.rl_rule), ptr(self.rl_rule, u8p), ptr(self.rl_value, i64p),
            self.n_quotas, ptr(self.quota_ns_str, u32p), ptr(self.quota_name_str, u32p), ptr(self.quota_item_off, u32p),
            len(self.qitem_type), ptr(self.qitem_type, u8p), ptr(self.qitem_value, i64p),
            self.n_endpoints, ptr(self.ep_ns_str, u32p), ptr(self.ep_name_str, u32p), ptr(self.ep_backend_off, u32p),
            len(self.backend_weight), ptr(self.backend_weight, i32p),
        )


def endpoint_backends(e, ready_backends=None):
    """(backend names, weights) of one ArksEndpoint in the order the controller emits HTTPRoute backendRefs
    (internal/controller/arksendpoint_controller.go:283-347): static routeConfigs, then ready Services at defaultWeight"""
    md = e["metadata"]
    ns = md.get("namespace", "default")
    names, weights = [], []
    spec = e.get("spec", {})
    for rc in spec.get("routeConfigs") or []:
        names.append(rc["name"])
        weights.append(int(rc.get("weight", 1)))  # Gateway API backendRef weight defaults to 1
    for svc in (ready_backends or {}).get((ns, md["name"]), []):
        if svc in names:
            continue
        names.append(svc)
        weights.append(int(spec.get("defaultWeight", 1)))
    return names, weights


def endpoint_pricing(e):
    """(prompt, completion) of an ArksEndpoint's optional spec.pricing: integer prices per token in the unit of the `cost` quota
    items (nano-dollars per token = dollars per 1M tokens x 1000); (0, 0) when absent. ValueError when a price is negative,
    not an integer or out of int64 range"""
    pr = (e.get("spec") or {}).get("pricing")
    if pr is None:
        return 0, 0
    if not isinstance(pr, dict):
        raise ValueError(f"spec.pricing must be an object, not {pr!r}")
    out = []
    for k in ("prompt", "completion"):
        v = pr.get(k, 0)
        if isinstance(v, bool) or not isinstance(v, int) or not 0 <= v < 2**63:
            raise ValueError(f"spec.pricing.{k} must be an integer in [0, 2^63), not {v!r}")
        out.append(v)
    return out[0], out[1]


def simple_token(name, namespace, token, model, limits, quota=""):
    """Convenience: one ArksToken with a single qos entry (limits: list of (type, value))."""
    return {"metadata": {"name": name, "namespace": namespace},
            "spec": {"token": token, "qos": [{"arksEndpoint": {"name": model},
                                             "rateLimits": [{"type": t, "value": v} for t, v in limits],
                                             "quota": {"name": quota}}]}}


def simple_quota(name, namespace, items):
    return {"metadata": {"name": name, "namespace": namespace},
            "spec": {"quotas": [{"type": t, "value": v} for t, v in items]}}


def simple_endpoint(name, namespace, default_weight=1, routes=(), pricing=None):
    e = {"metadata": {"name": name, "namespace": namespace},
         "spec": {"defaultWeight": default_weight,
                  "routeConfigs": [{"name": n, "weight": w} for n, w in routes]}}
    if pricing is not None:
        e["spec"]["pricing"] = {"prompt": pricing[0], "completion": pricing[1]}
    return e
