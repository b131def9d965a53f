// Object-level config plane (host only, no CUDA): the objects behind arks_upsert_* / arks_delete_*.
//
// Reference: the gateway's qosconfig.ConfigProvider is an informer cache over three CRDs, keyed by namespace/name
// (pkg/gateway/qosconfig/arks_impl.go:104-189: AddEventHandler on ArksToken / ArksQuota / ArksEndpoint; lookups at :300-340).
// One informer event = one call here, O(that object). flatten() lays the store out as the arks_tables the device image is
// built from (include/arks_gateway.h) — objects in (namespace, name) order, so the image is a pure function of the store.
#pragma once
#include <cstdint>
#include <map>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/arks_gateway.h"

namespace arks {

struct FlatTables {
  std::vector<uint8_t> bytes;
  std::vector<uint32_t> off{0};
  std::vector<uint32_t> tok_token, tok_ns, tok_name, tok_qos_off{0}, qos_model, qos_rl_off{0}, quota_ns, quota_name, quota_item_off{0};
  std::vector<uint32_t> ep_ns, ep_name, ep_off{0};
  std::vector<int32_t> qos_quota, bw;
  std::vector<uint8_t> rl_rule, qi_type;
  std::vector<int64_t> rl_value, qi_value;
  std::unordered_map<std::string, uint32_t> seen;

  uint32_t str(const std::string& s) {
    auto it = seen.find(s);
    if (it != seen.end()) return it->second;
    bytes.insert(bytes.end(), s.begin(), s.end());
    off.push_back((uint32_t)bytes.size());
    return seen.emplace(s, (uint32_t)off.size() - 2).first->second;
  }
  // pointers into this object: valid while it lives and is not modified
  arks_tables view() const {
    static const uint64_t zero[2] = {0, 0};  // what an empty array points at (never read: its count is 0)
    auto P = [&](const auto& v) { return v.empty() ? reinterpret_cast<decltype(v.data())>(zero) : v.data(); };
    arks_tables t{};
    t.str_bytes = P(bytes);
    t.str_off = off.data();
    t.n_str = (uint32_t)off.size() - 1;
    t.n_tokens = (uint32_t)tok_token.size();
    t.tok_token_str = P(tok_token);
    t.tok_ns_str = P(tok_ns);
    t.tok_name_str = P(tok_name);
    t.tok_qos_off = tok_qos_off.data();
    t.n_qos = (uint32_t)qos_model.size();
    t.qos_model_str = P(qos_model);
    t.qos_quota = P(qos_quota);
    t.qos_rl_off = qos_rl_off.data();
    t.n_rl = (uint32_t)rl_rule.size();
    t.rl_rule = P(rl_rule);
    t.rl_value = P(rl_value);
    t.n_quotas = (uint32_t)quota_ns.size();
    t.quota_ns_str = P(quota_ns);
    t.quota_name_str = P(quota_name);
    t.quota_item_off = quota_item_off.data();
    t.n_qitems = (uint32_t)qi_type.size();
    t.qitem_type = P(qi_type);
    t.qitem_value = P(qi_value);
    t.n_endpoints = (uint32_t)ep_ns.size();
    t.ep_ns_str = P(ep_ns);
    t.ep_name_str = P(ep_name);
    t.ep_backend_off = ep_off.data();
    t.n_backends = (uint32_t)bw.size();
    t.backend_weight = P(bw);
    return t;
  }
};

// Shape check of a caller-built snapshot (arks_prepare_tables / arks_load_tables): every index the host code and the kernels
// will follow must stay inside its array. The reference gets its objects from the API server, validated by the CRD schemas
// (api/v1/*_types.go kubebuilder markers); a C caller has no such guard, and a bad offset here would be an out-of-bounds read
// on the device. Returns NULL when the snapshot is well formed, else what is wrong (static text).
inline const char* tables_shape_error(const arks_tables* t) {
  if (!t) return "null tables";
  auto csr = [](const uint32_t* off, uint32_t n, uint32_t total) {
    if (!off || off[0] != 0 || off[n] != total) return false;
    for (uint32_t i = 0; i < n; i++)
      if (off[i] > off[i + 1]) return false;
    return true;
  };
  auto ids = [&](const uint32_t* id, uint32_t n) {
    if (n && !id) return false;
    for (uint32_t i = 0; i < n; i++)
      if (id[i] >= t->n_str) return false;
    return true;
  };
  if (!t->str_off || (t->n_str && t->str_off[t->n_str] && !t->str_bytes)) return "string pool: null pointer";
  for (uint32_t i = 0; i < t->n_str; i++)
    if (t->str_off[i] > t->str_off[i + 1]) return "string pool: offsets decrease";
  if (!ids(t->tok_token_str, t->n_tokens) || !ids(t->tok_ns_str, t->n_tokens) || !ids(t->tok_name_str, t->n_tokens))
    return "ArksToken: string id out of range";
  if (!csr(t->tok_qos_off, t->n_tokens, t->n_qos)) return "tok_qos_off is not a CSR over the qos entries";
  if (!ids(t->qos_model_str, t->n_qos)) return "qos: model string id out of range";
  if (t->n_qos && !t->qos_quota) return "qos_quota: null pointer";
  if (!csr(t->qos_rl_off, t->n_qos, t->n_rl)) return "qos_rl_off is not a CSR over the rate limits";
  if (t->n_rl && (!t->rl_rule || !t->rl_value)) return "rate limits: null pointer";
  if (!ids(t->quota_ns_str, t->n_quotas) || !ids(t->quota_name_str, t->n_quotas)) return "ArksQuota: string id out of range";
  if (!csr(t->quota_item_off, t->n_quotas, t->n_qitems)) return "quota_item_off is not a CSR over the quota items";
  if (t->n_qitems && (!t->qitem_type || !t->qitem_value)) return "quota items: null pointer";
  for (uint32_t i = 0; i < t->n_rl; i++)
    if (t->rl_rule[i] >= ARKS_N_RULES) return "unknown rate-limit rule";
  for (uint32_t i = 0; i < t->n_qitems; i++)
    if (t->qitem_type[i] > ARKS_QT_COST) return "unknown quota type";
  if (!ids(t->ep_ns_str, t->n_endpoints) || !ids(t->ep_name_str, t->n_endpoints)) return "ArksEndpoint: string id out of range";
  if (!csr(t->ep_backend_off, t->n_endpoints, t->n_backends)) return "ep_backend_off is not a CSR over the backends";
  if (t->n_backends && !t->backend_weight) return "backend_weight: null pointer";
  for (uint32_t i = 0; i < t->n_backends; i++)
    if (t->backend_weight[i] < 0) return "negative backend weight";
  return nullptr;
}

struct ConfigStore {
  using Key = std::pair<std::string, std::string>;  // (namespace, name)
  struct Qos {
    std::string model, quota;
    std::vector<uint8_t> rl_rule;
    std::vector<int64_t> rl_value;
  };
  struct Token {
    std::string token;
    std::vector<Qos> qos;
  };
  struct Quota {
    std::vector<uint8_t> type;
    std::vector<int64_t> value;
  };
  std::map<Key, Token> tokens;
  std::map<Key, Quota> quotas;
  std::map<Key, std::vector<int32_t>> endpoints;

  static Key key(const char* ns, uint32_t ns_len, const char* name, uint32_t name_len) {
    return {std::string(ns ? ns : "", ns_len), std::string(name ? name : "", name_len)};
  }
  void upsert_token(const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const char* token, uint32_t token_len,
                    const arks_qos_spec* qos, uint32_t n_qos) {
    Token t;
    t.token.assign(token ? token : "", token_len);
    for (uint32_t i = 0; i < n_qos; i++) {
      Qos q;
      q.model.assign(qos[i].model ? qos[i].model : "", qos[i].model_len);
      q.quota.assign(qos[i].quota ? qos[i].quota : "", qos[i].quota_len);
      if (qos[i].n_rl) {
        q.rl_rule.assign(qos[i].rl_rule, qos[i].rl_rule + qos[i].n_rl);
        q.rl_value.assign(qos[i].rl_value, qos[i].rl_value + qos[i].n_rl);
      }
      t.qos.push_back(std::move(q));
    }
    tokens[key(ns, ns_len, name, name_len)] = std::move(t);
  }
  void upsert_quota(const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const uint8_t* type, const int64_t* value,
                    uint32_t n) {
    Quota q;
    if (n) {
      q.type.assign(type, type + n);
      q.value.assign(value, value + n);
    }
    quotas[key(ns, ns_len, name, name_len)] = std::move(q);
  }
  void upsert_endpoint(const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const int32_t* w, uint32_t n) {
    std::vector<int32_t>& v = endpoints[key(ns, ns_len, name, name_len)];
    v.clear();
    if (n) v.assign(w, w + n);
  }
  // which: 0 token, 1 quota, 2 endpoint; false when the object is not there
  bool erase(int which, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len) {
    const Key k = key(ns, ns_len, name, name_len);
    return which == 0 ? tokens.erase(k) != 0 : which == 1 ? quotas.erase(k) != 0 : endpoints.erase(k) != 0;
  }

  void flatten(FlatTables* f) const {
    std::map<Key, int32_t> quota_index;
    for (const auto& kv : quotas) {
      quota_index.emplace(kv.first, (int32_t)f->quota_ns.size());
      f->quota_ns.push_back(f->str(kv.first.first));
      f->quota_name.push_back(f->str(kv.first.second));
      f->qi_type.insert(f->qi_type.end(), kv.second.type.begin(), kv.second.type.end());
      f->qi_value.insert(f->qi_value.end(), kv.second.value.begin(), kv.second.value.end());
      f->quota_item_off.push_back((uint32_t)f->qi_type.size());
    }
    for (const auto& kv : tokens) {
      f->tok_token.push_back(f->str(kv.second.token));
      f->tok_ns.push_back(f->str(kv.first.first));
      f->tok_name.push_back(f->str(kv.first.second));
      for (const Qos& q : kv.second.qos) {
        f->qos_model.push_back(f->str(q.model));
        int32_t qi = ARKS_QUOTA_NONE;  // quota.name == "" (handle_request.go:185)
        if (!q.quota.empty()) {        // the ArksQuota of the token's own namespace (check.go:76-84); absent -> 500 at request time
          auto it = quota_index.find({kv.first.first, q.quota});
          qi = it == quota_index.end() ? ARKS_QUOTA_MISSING : it->second;
        }
        f->qos_quota.push_back(qi);
        f->rl_rule.insert(f->rl_rule.end(), q.rl_rule.begin(), q.rl_rule.end());
        f->rl_value.insert(f->rl_value.end(), q.rl_value.begin(), q.rl_value.end());
        f->qos_rl_off.push_back((uint32_t)f->rl_rule.size());
      }
      f->tok_qos_off.push_back((uint32_t)f->qos_model.size());
    }
    for (const auto& kv : endpoints) {
      f->ep_ns.push_back(f->str(kv.first.first));
      f->ep_name.push_back(f->str(kv.first.second));
      f->bw.insert(f->bw.end(), kv.second.begin(), kv.second.end());
      f->ep_off.push_back((uint32_t)f->bw.size());
    }
  }
};

}  // namespace arks
