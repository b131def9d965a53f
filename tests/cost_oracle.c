/* cost_oracle.c — TEST-ONLY: the CPU oracle (oracle/ork_core.c, compiled in here unchanged) with pricing-based quotas: the
 * `cost` quota item (ARKS_QT_COST) and per-endpoint prices (include/arks_gateway.h arks_set_endpoint_price).
 *
 * The statement is Redis's: every ArksQuota gets a fourth key, its cost usage, next to the prompt / response / total keys.
 * The core oracle refuses item type 3, so it is handed the tables with the cost items taken out; this file keeps them (their
 * spec index and limit per quota) and:
 *   - decides row by row: after the core oracle's decision of a row that reached the quota check, the first over-limit item
 *     in spec order over ALL items (cost ones included) is the row's answer. A row the core admitted but a cost item denies
 *     gives back its request-type increments and its pre-charge entries (they were the row's own, on the same keys);
 *   - bills every counted response row prompt x p_prompt + completion x p_completion per cost item, and metered rows (N5)
 *     their count at the side's price, all modulo 2^64;
 *   - resolves each qos entry's price at create / reload from the price map as it is then (the endpoint its (token
 *     namespace, model) resolves to; none: 0), and carries the cost key by (namespace, quotaName);
 *   - syncs the four columns in one pass (ork_sync_quota_usage's rule, over the cost column too).
 * Built as its own library (tests/_build/libarks_oracle_cost.so) next to ork_json.c. */
#define ork_create ork_create_plain
#define ork_request_batch ork_request_batch_plain
#define ork_response_batch ork_response_batch_plain
#define ork_reload ork_reload_plain
#define ork_destroy ork_destroy_plain
#include "../oracle/ork_core.c"
#undef ork_create
#undef ork_request_batch
#undef ork_response_batch
#undef ork_reload
#undef ork_destroy

ork* ork_create(const arks_tables* t);
int ork_request_batch(ork* o, const arks_request_batch* b, arks_request_result* r);
int ork_response_batch(ork* o, const arks_response_batch* b, arks_response_result* r);
int ork_reload(ork* o, const arks_tables* t);
void ork_destroy(ork* o);
int ork_set_endpoint_price(ork* o, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, int64_t prompt, int64_t completion);
int ork_snapshot_quota_cost(ork* o, int64_t* cost);
void ork_meter_charge(ork* o, uint32_t n, const int32_t* qos, const int64_t* count, int side, int64_t now);
int ork_sync_quota_usage4(ork* o, uint32_t q, uint32_t* status_present, int64_t status_used[4], int restore);

/* the price map (namespace \0 name -> prices), process-wide: one oracle per test at a time is what the tests use, but the
 * per-oracle state below is keyed by the oracle like sliding_oracle.c's */
typedef struct {
  char key[600];
  int64_t p[2];
} price_ent;
typedef struct {
  const ork* o;
  uint32_t n_quotas, n_qos;
  int64_t* cost;        /* n_quotas: the fourth key */
  uint32_t* c_off;      /* n_quotas + 1: CSR into c_index / c_limit */
  uint8_t* c_index;     /* spec index of the cost item inside its quota */
  int64_t* c_limit;
  uint8_t* keep_index;  /* per quota, spec index of each item the core oracle kept (its detail -> the spec index) */
  uint32_t* keep_off;
  int64_t* price;       /* n_qos * 2 */
  price_ent* prices;
  uint32_t n_prices, cap_prices;
} side;
static side g_side[16];

static side* side_of(const ork* o) {
  for (int k = 0; k < 16; k++)
    if (g_side[k].o == o) return &g_side[k];
  for (int k = 0; k < 16; k++)
    if (!g_side[k].o) {
      memset(&g_side[k], 0, sizeof g_side[k]);
      g_side[k].o = o;
      return &g_side[k];
    }
  return NULL;
}

static void key2(char* out, size_t cap, const uint8_t* a, size_t al, const uint8_t* b, size_t bl) {
  memset(out, 0, cap);
  if (al + bl + 2 > cap) return;
  memcpy(out, a, al);
  memcpy(out + al + 1, b, bl);
}

/* the tables without their cost items (what the core oracle accepts), plus the side's item lists */
typedef struct {
  arks_tables t;
  uint32_t* off;
  uint8_t* type;
  int64_t* value;
} stripped;
static int strip(const arks_tables* t, stripped* s, side* sd) {
  s->t = *t;
  s->off = (uint32_t*)calloc((size_t)t->n_quotas + 1, 4);
  s->type = (uint8_t*)malloc((size_t)t->n_qitems + 1);
  s->value = (int64_t*)malloc(8 * (size_t)t->n_qitems + 8);
  free(sd->c_off); free(sd->c_index); free(sd->c_limit); free(sd->keep_index); free(sd->keep_off);
  sd->c_off = (uint32_t*)calloc((size_t)t->n_quotas + 1, 4);
  sd->keep_off = (uint32_t*)calloc((size_t)t->n_quotas + 1, 4);
  sd->c_index = (uint8_t*)malloc((size_t)t->n_qitems + 1);
  sd->c_limit = (int64_t*)malloc(8 * (size_t)t->n_qitems + 8);
  sd->keep_index = (uint8_t*)malloc((size_t)t->n_qitems + 1);
  uint32_t nk = 0, nc = 0;
  for (uint32_t q = 0; q < t->n_quotas; q++) {
    for (uint32_t j = t->quota_item_off[q]; j < t->quota_item_off[q + 1]; j++) {
      if (t->qitem_type[j] > ARKS_QT_COST) return ARKS_E_BAD_TABLE;
      const uint8_t idx = (uint8_t)(j - t->quota_item_off[q]);
      if (t->qitem_type[j] == ARKS_QT_COST) {
        sd->c_index[nc] = idx;
        sd->c_limit[nc++] = t->qitem_value[j];
      } else {
        s->type[nk] = t->qitem_type[j];
        s->value[nk] = t->qitem_value[j];
        sd->keep_index[nk++] = idx;
      }
    }
    s->off[q + 1] = nk;
    sd->c_off[q + 1] = nc;
    sd->keep_off[q + 1] = nk;
  }
  s->t.quota_item_off = s->off;
  s->t.qitem_type = s->type;
  s->t.qitem_value = s->value;
  s->t.n_qitems = nk;
  return 0;
}
static void strip_free(stripped* s) {
  free(s->off); free(s->type); free(s->value);
}

/* each qos entry's price: the endpoint its (token namespace, model) resolves to, as priced now */
static void resolve_prices(const ork* o, side* sd) {
  free(sd->price);
  sd->n_qos = o->n_qos;
  sd->price = (int64_t*)calloc(2 * (size_t)o->n_qos + 2, 8);
  for (uint32_t q = 0; q < o->n_qos; q++) {
    size_t ml, nl, el;
    const uint8_t* m = S(o, o->qos_model_str[q], &ml);
    const int32_t ep = find_endpoint(o, o->tok_ns_str[o->qos_token[q]], m, ml);
    if (ep < 0) continue;
    const uint8_t* ns = S(o, o->ep_ns_str[ep], &nl);
    const uint8_t* nm = S(o, o->ep_name_str[ep], &el);
    char k[600];
    key2(k, sizeof k, ns, nl, nm, el);
    for (uint32_t p = 0; p < sd->n_prices; p++)
      if (!memcmp(sd->prices[p].key, k, sizeof k)) {
        sd->price[2 * (size_t)q] = sd->prices[p].p[0];
        sd->price[2 * (size_t)q + 1] = sd->prices[p].p[1];
      }
  }
}

ork* ork_create(const arks_tables* t) {
  side tmp;
  memset(&tmp, 0, sizeof tmp);
  stripped s;
  if (strip(t, &s, &tmp)) {
    strip_free(&s);
    free(tmp.c_off); free(tmp.c_index); free(tmp.c_limit); free(tmp.keep_index); free(tmp.keep_off);
    return NULL;
  }
  ork* o = ork_create_plain(&s.t);
  strip_free(&s);
  side* sd = o ? side_of(o) : NULL;
  if (!sd) {
    free(tmp.c_off); free(tmp.c_index); free(tmp.c_limit); free(tmp.keep_index); free(tmp.keep_off);
    if (o) ork_destroy_plain(o);
    return NULL;
  }
  tmp.o = o;
  *sd = tmp;
  sd->n_quotas = o->n_quotas;
  sd->cost = (int64_t*)calloc((size_t)o->n_quotas + 1, 8);
  resolve_prices(o, sd);
  return o;
}

void ork_destroy(ork* o) {
  side* sd = side_of(o);
  if (sd) {
    free(sd->cost); free(sd->c_off); free(sd->c_index); free(sd->c_limit); free(sd->keep_index); free(sd->keep_off);
    free(sd->price); free(sd->prices);
    memset(sd, 0, sizeof *sd);
  }
  ork_destroy_plain(o);
}

int ork_set_endpoint_price(ork* o, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, int64_t prompt, int64_t completion) {
  if (prompt < 0 || completion < 0) return ARKS_E_INVALID_ARG;
  side* sd = side_of(o);
  char k[600];
  key2(k, sizeof k, (const uint8_t*)ns, ns_len, (const uint8_t*)name, name_len);
  for (uint32_t p = 0; p < sd->n_prices; p++)
    if (!memcmp(sd->prices[p].key, k, sizeof k)) {
      sd->prices[p].p[0] = prompt;
      sd->prices[p].p[1] = completion;
      return 0;
    }
  if (sd->n_prices == sd->cap_prices) {
    sd->cap_prices = sd->cap_prices ? 2 * sd->cap_prices : 64;
    sd->prices = (price_ent*)realloc(sd->prices, sd->cap_prices * sizeof *sd->prices);
  }
  memcpy(sd->prices[sd->n_prices].key, k, sizeof k);
  sd->prices[sd->n_prices].p[0] = prompt;
  sd->prices[sd->n_prices].p[1] = completion;
  sd->n_prices++;
  return 0;
}

int ork_reload(ork* o, const arks_tables* t) {
  side* sd = side_of(o);
  side next = *sd;
  next.c_off = NULL; next.c_index = NULL; next.c_limit = NULL; next.keep_index = NULL; next.keep_off = NULL;
  stripped s;
  int rc = strip(t, &s, &next);
  if (!rc) {
    /* the old quota keys, to carry the cost key by (namespace, quotaName) */
    const uint32_t n_old = o->n_quotas;
    char(*old_keys)[600] = malloc(((size_t)n_old + 1) * 600);
    for (uint32_t q = 0; q < n_old; q++) {
      size_t a, b;
      const uint8_t* ns = S(o, o->quota_ns_str[q], &a);
      const uint8_t* nm = S(o, o->quota_name_str[q], &b);
      key2(old_keys[q], 600, ns, a, nm, b);
    }
    const int precharge = o->precharge; /* a switch of the context: the core's reload starts from a fresh oracle */
    rc = ork_reload_plain(o, &s.t);
    if (!rc) {
      o->precharge = precharge;
      int64_t* cost = (int64_t*)calloc((size_t)o->n_quotas + 1, 8);
      for (uint32_t q = 0; q < o->n_quotas; q++) {
        size_t a, b;
        const uint8_t* ns = S(o, o->quota_ns_str[q], &a);
        const uint8_t* nm = S(o, o->quota_name_str[q], &b);
        char k[600];
        key2(k, sizeof k, ns, a, nm, b);
        for (uint32_t p = 0; p < n_old; p++)
          if (!memcmp(k, old_keys[p], 600)) {
            cost[q] = sd->cost[p];
            break;
          }
      }
      free(sd->cost); free(sd->c_off); free(sd->c_index); free(sd->c_limit); free(sd->keep_index); free(sd->keep_off);
      next.cost = cost;
      next.n_quotas = o->n_quotas;
      *sd = next;
      resolve_prices(o, sd);
    }
    free(old_keys);
  }
  strip_free(&s);
  if (rc) {
    free(next.c_off); free(next.c_index); free(next.c_limit); free(next.keep_index); free(next.keep_off);
  }
  return rc;
}

int ork_request_batch(ork* o, const arks_request_batch* b, arks_request_result* r) {
  int rc = check_time(o, b->now_unix);
  if (rc) return rc;
  side* sd = side_of(o);
  for (uint32_t i = 0; i < b->n; i++) {
    const uint32_t pc_before = o->pc_n;
    handle_request(o, b, r, i, i);
    const uint8_t reason = r->reason[i];
    if (reason != ARKS_R_OK && reason != ARKS_R_QUOTA) continue;
    const int32_t q = r->qos[i];
    const int32_t qt = q >= 0 ? o->qos_quota[q] : -1;
    if (qt < 0) continue;
    /* the core's answer as a spec index (255: admitted), then the first over-limit cost item before it */
    const uint32_t k0 = sd->keep_off[qt];
    uint32_t first = reason == ARKS_R_QUOTA ? sd->keep_index[k0 + r->detail[i]] : 255u;
    int64_t cur = r->cur_usage[i], lim = r->limit_max[i];
    for (uint32_t c = sd->c_off[qt]; c < sd->c_off[qt + 1]; c++)
      if (sd->c_index[c] < first && sd->cost[qt] > sd->c_limit[c]) {
        first = sd->c_index[c];
        cur = sd->cost[qt];
        lim = sd->c_limit[c];
        break;
      }
    if (first == 255u) continue;
    if (reason == ARKS_R_OK) { /* admitted by the core, denied by a cost item: the row's own increments go back */
      for (uint32_t j = o->qos_rl_off[q]; j < o->qos_rl_off[q + 1]; j++) {
        const int rule = o->rl_rule[j];
        if (RULE_IS_REQUEST[rule]) rate_incr(o, (uint32_t)q, rule, ork_window_start(b->now_unix, rule), -1);
      }
      o->pc_n = pc_before;
      r->flags[i] = 0;
      r->pick[i] = -1;
    }
    r->reason[i] = ARKS_R_QUOTA;
    r->detail[i] = (uint8_t)first;
    r->cur_usage[i] = cur;
    r->limit_max[i] = lim;
  }
  for (uint32_t k = 0; k < o->pc_n; k++) rate_incr(o, o->pc[k].q, o->pc[k].rule, ork_window_start(b->now_unix, o->pc[k].rule), o->pc[k].amount);
  o->pc_n = 0;
  o->est = NULL;
  o->est_n = 0;
  return 0;
}

int ork_response_batch(ork* o, const arks_response_batch* b, arks_response_result* r) {
  const int rc = ork_response_batch_plain(o, b, r);
  if (rc) return rc;
  side* sd = side_of(o);
  for (uint32_t i = 0; i < b->n; i++) {
    if (!r->counted[i] || r->reason[i] == ARKS_R_QUOTA_CONFIG_RESP || r->reason[i] == ARKS_R_QOS_GONE) continue;
    const int32_t q = b->qos[i], qt = o->qos_quota[q];
    if (qt < 0) continue;
    const uint64_t n = sd->c_off[qt + 1] - sd->c_off[qt];
    const uint64_t add = ((uint64_t)r->usage[3 * (size_t)i] * (uint64_t)sd->price[2 * (size_t)q] +
                          (uint64_t)r->usage[3 * (size_t)i + 1] * (uint64_t)sd->price[2 * (size_t)q + 1]) * n;
    sd->cost[qt] = (int64_t)((uint64_t)sd->cost[qt] + add);
  }
  return 0;
}

/* N5: metered rows billed `count` each (side 0 a prompt, 1 a completion chunk): tpm / tpd per entry, the side's quota item and
 * total per item, gateway_token_usage of the side, the cost key at the side's price per cost item */
void ork_meter_charge(ork* o, uint32_t n, const int32_t* qos, const int64_t* count, int side_, int64_t now) {
  side* sd = side_of(o);
  for (uint32_t i = 0; i < n; i++) {
    const int32_t q = qos[i];
    const int64_t c = count[i];
    if (q < 0 || (uint32_t)q >= o->n_qos || c == 0) continue;
    for (uint32_t j = o->qos_rl_off[q]; j < o->qos_rl_off[q + 1]; j++)
      if (!RULE_IS_REQUEST[o->rl_rule[j]]) rate_incr(o, (uint32_t)q, o->rl_rule[j], ork_window_start(now, o->rl_rule[j]), c);
    o->metrics[(size_t)q * ARKS_METRIC_COLS + ARKS_METRIC_USAGE + side_] += c;
    const int32_t qt = o->qos_quota[q];
    if (qt < 0) continue;
    for (uint32_t j = o->quota_item_off[qt]; j < o->quota_item_off[qt + 1]; j++) {
      const int ty = o->qitem_type[j];
      if (ty == side_ || ty == ARKS_QT_TOTAL) o->quota_use[(size_t)qt * 3 + ty] = (int64_t)((uint64_t)o->quota_use[(size_t)qt * 3 + ty] + (uint64_t)c);
    }
    const uint64_t nc = sd->c_off[qt + 1] - sd->c_off[qt];
    sd->cost[qt] = (int64_t)((uint64_t)sd->cost[qt] + (uint64_t)c * (uint64_t)sd->price[2 * (size_t)q + side_] * nc);
  }
}

int ork_snapshot_quota_cost(ork* o, int64_t* cost) {
  const side* sd = side_of(o);
  memcpy(cost, sd->cost, 8 * (size_t)o->n_quotas);
  return 0;
}

/* syncQuotaUsage over the four keys of quota q (ork_sync_quota_usage's rule, arks_impl.go:226-296) */
int ork_sync_quota_usage4(ork* o, uint32_t q, uint32_t* status_present, int64_t status_used[4], int restore) {
  if (q >= o->n_quotas) return ARKS_E_INVALID_ARG;
  side* sd = side_of(o);
  int64_t* key[4] = {&o->quota_use[(size_t)q * 3], &o->quota_use[(size_t)q * 3 + 1], &o->quota_use[(size_t)q * 3 + 2], &sd->cost[q]};
  /* the items in spec order: the kept ones and the cost ones merged by spec index */
  uint8_t ty[256];
  const uint32_t nk = sd->keep_off[q + 1] - sd->keep_off[q], nc = sd->c_off[q + 1] - sd->c_off[q];
  for (uint32_t k = 0; k < nk; k++) ty[sd->keep_index[sd->keep_off[q] + k]] = o->qitem_type[o->quota_item_off[q] + k];
  for (uint32_t c = 0; c < nc; c++) ty[sd->c_index[sd->c_off[q] + c]] = ARKS_QT_COST;
  int update_cr = 0, update_quota = 0;
  for (uint32_t j = 0; j < nk + nc; j++) {
    const int t = ty[j];
    if (*status_present & (1u << t)) {
      if (status_used[t] < *key[t]) { update_cr = 1; status_used[t] = *key[t]; }
      else if (status_used[t] > *key[t]) update_quota = 1;
    } else {
      update_cr = 1; *status_present |= 1u << t; status_used[t] = *key[t];
    }
  }
  if (update_quota)
    for (uint32_t j = 0; j < nk + nc; j++) {
      const int t = ty[j];
      if (!restore) *key[t] = 0;
      else if (status_used[t] > *key[t]) *key[t] = status_used[t];
    }
  return update_cr | update_quota << 1;
}
