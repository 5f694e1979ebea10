// K0 (compat): host-side clone of CPython's `random` module (MT19937) and of the three
// reference samplers that consume it.  Bit exact with CPython 3.12's Lib/random.py +
// Modules/_randommodule.c; the reference call sites are cited per function in qrec.h.
//
// The MT19937 stream is serial by construction, so this stays on one host thread; the
// throughput path uses the device Philox sampler (sampler_philox.cu) instead.
#include <cstring>
#include <vector>

#include "common.h"

namespace {

constexpr int N = 624, M = 397;
constexpr uint32_t MATRIX_A = 0x9908b0dfu, UPPER = 0x80000000u, LOWER = 0x7fffffffu;

inline void init_genrand(qrec_mt19937* st, uint32_t s) {
  uint32_t* mt = st->mt;
  mt[0] = s;
  for (int k = 1; k < N; ++k) mt[k] = 1812433253u * (mt[k - 1] ^ (mt[k - 1] >> 30)) + (uint32_t)k;
  st->index = N;
}

void init_by_array(qrec_mt19937* st, const uint32_t* key, size_t len) {
  uint32_t* mt = st->mt;
  init_genrand(st, 19650218u);
  size_t i = 1, j = 0;
  size_t k = (N > len ? (size_t)N : len);
  for (; k; --k) {
    mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1664525u)) + key[j] + (uint32_t)j;
    ++i; ++j;
    if (i >= (size_t)N) { mt[0] = mt[N - 1]; i = 1; }
    if (j >= len) j = 0;
  }
  for (k = N - 1; k; --k) {
    mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1566083941u)) - (uint32_t)i;
    ++i;
    if (i >= (size_t)N) { mt[0] = mt[N - 1]; i = 1; }
  }
  mt[0] = 0x80000000u;
}

inline void regenerate(qrec_mt19937* st) {
  uint32_t* mt = st->mt;
  int kk = 0;
  uint32_t y;
  for (; kk < N - M; ++kk) {
    y = (mt[kk] & UPPER) | (mt[kk + 1] & LOWER);
    mt[kk] = mt[kk + M] ^ (y >> 1) ^ ((y & 1u) ? MATRIX_A : 0u);
  }
  for (; kk < N - 1; ++kk) {
    y = (mt[kk] & UPPER) | (mt[kk + 1] & LOWER);
    mt[kk] = mt[kk + (M - N)] ^ (y >> 1) ^ ((y & 1u) ? MATRIX_A : 0u);
  }
  y = (mt[N - 1] & UPPER) | (mt[0] & LOWER);
  mt[N - 1] = mt[M - 1] ^ (y >> 1) ^ ((y & 1u) ? MATRIX_A : 0u);
  st->index = 0;
}

inline uint32_t next_u32(qrec_mt19937* st) {
  if (st->index >= (uint32_t)N) regenerate(st);
  uint32_t y = st->mt[st->index++];
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}

// Random._randbelow_with_getrandbits: k = n.bit_length(); r = getrandbits(k) until r < n,
// with getrandbits(k <= 32) = genrand_uint32() >> (32 - k).
inline uint32_t randbelow(qrec_mt19937* st, uint32_t n) {
  const int k = 32 - __builtin_clz(n);  // n >= 1
  const int sh = 32 - k;
  uint32_t r = next_u32(st) >> sh;
  while (r >= n) r = next_u32(st) >> sh;
  return r;
}

inline bool row_contains(const int64_t* rowptr, const int32_t* cols, int32_t row, int32_t x) {
  int64_t lo = rowptr[row], hi = rowptr[row + 1];
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    const int32_t c = cols[mid];
    if (c < x) lo = mid + 1;
    else if (c > x) hi = mid;
    else return true;
  }
  return false;
}

}  // namespace

extern "C" {

int qrec_mt_seed(qrec_mt19937* st, uint64_t seed) {
  QREC_REQUIRE(st != nullptr, "qrec_mt_seed: null state");
  uint32_t key[2] = {(uint32_t)(seed & 0xffffffffu), (uint32_t)(seed >> 32)};
  init_by_array(st, key, key[1] ? 2 : 1);
  return QREC_OK;
}

int qrec_mt_set_state(qrec_mt19937* st, const uint32_t* s) {
  QREC_REQUIRE(st && s, "qrec_mt_set_state: null pointer");
  QREC_REQUIRE(s[624] <= 624u, "qrec_mt_set_state: index %u out of range", s[624]);
  std::memcpy(st->mt, s, sizeof(uint32_t) * N);
  st->index = s[624];
  return QREC_OK;
}

int qrec_mt_get_state(const qrec_mt19937* st, uint32_t* s) {
  QREC_REQUIRE(st && s, "qrec_mt_get_state: null pointer");
  std::memcpy(s, st->mt, sizeof(uint32_t) * N);
  s[624] = st->index;
  return QREC_OK;
}

uint32_t qrec_mt_next_u32(qrec_mt19937* st) { return next_u32(st); }

double qrec_mt_random(qrec_mt19937* st) {
  const uint32_t a = next_u32(st) >> 5, b = next_u32(st) >> 6;
  return (a * 67108864.0 + b) * (1.0 / 9007199254740992.0);
}

uint32_t qrec_mt_randbelow(qrec_mt19937* st, uint32_t n) { return n ? randbelow(st, n) : 0u; }

int qrec_mt_shuffle_i32(qrec_mt19937* st, int64_t n, int32_t* x) {
  QREC_REQUIRE(st && (x || n == 0), "qrec_mt_shuffle_i32: null pointer");
  QREC_REQUIRE(n >= 0 && n <= 0x7fffffffLL, "qrec_mt_shuffle_i32: n=%lld out of range", (long long)n);
  for (int64_t k = n - 1; k >= 1; --k) {
    const uint32_t r = randbelow(st, (uint32_t)(k + 1));
    const int32_t t = x[k]; x[k] = x[r]; x[r] = t;
  }
  return QREC_OK;
}

int qrec_mt_shuffle_pairs_i32(qrec_mt19937* st, int64_t n, int32_t* a, int32_t* b) {
  QREC_REQUIRE(st && ((a && b) || n == 0), "qrec_mt_shuffle_pairs_i32: null pointer");
  QREC_REQUIRE(n >= 0 && n <= 0x7fffffffLL, "qrec_mt_shuffle_pairs_i32: n=%lld out of range", (long long)n);
  for (int64_t k = n - 1; k >= 1; --k) {
    const uint32_t r = randbelow(st, (uint32_t)(k + 1));
    int32_t t = a[k]; a[k] = a[r]; a[r] = t;
    t = b[k]; b[k] = b[r]; b[r] = t;
  }
  return QREC_OK;
}

int qrec_mt_data_split(qrec_mt19937* st, int64_t n, double test_ratio, uint8_t* keep) {
  QREC_REQUIRE(st && (keep || n == 0), "qrec_mt_data_split: null pointer");
  if (test_ratio >= 1 || test_ratio <= 0) test_ratio = 0.3;  // util/dataSplit.py:10-11
  for (int64_t k = 0; k < n; ++k) keep[k] = qrec_mt_random(st) < test_ratio ? 0 : 1;
  return QREC_OK;
}

int qrec_sample_bpr_epoch(qrec_mt19937* st, int32_t n_users, int32_t num_items,
                          const int64_t* pos_rowptr, const int32_t* pos_cols,
                          const int64_t* sorted_rowptr, const int32_t* sorted_cols,
                          int32_t* out_u, int32_t* out_i, int32_t* out_j) {
  QREC_REQUIRE(st && pos_rowptr && sorted_rowptr, "qrec_sample_bpr_epoch: null pointer");
  QREC_REQUIRE(n_users >= 0 && num_items >= 1, "qrec_sample_bpr_epoch: bad sizes");
  int64_t k = 0;
  for (int32_t u = 0; u < n_users; ++u) {
    const int64_t deg = sorted_rowptr[u + 1] - sorted_rowptr[u];
    QREC_REQUIRE(deg < num_items, "qrec_sample_bpr_epoch: user %d rated every item", u);
    for (int64_t p = pos_rowptr[u]; p < pos_rowptr[u + 1]; ++p) {
      uint32_t j = randbelow(st, (uint32_t)num_items);
      while (row_contains(sorted_rowptr, sorted_cols, u, (int32_t)j)) j = randbelow(st, (uint32_t)num_items);
      out_u[k] = u; out_i[k] = pos_cols[p]; out_j[k] = (int32_t)j;
      ++k;
    }
  }
  return QREC_OK;
}

int qrec_sample_pairwise(qrec_mt19937* st, int64_t n, int32_t num_items, const int32_t* u,
                         const int64_t* sorted_rowptr, const int32_t* sorted_cols, int32_t* out_j) {
  QREC_REQUIRE(st && sorted_rowptr && (n == 0 || (u && out_j)), "qrec_sample_pairwise: null pointer");
  QREC_REQUIRE(num_items >= 1, "qrec_sample_pairwise: num_items < 1");
  for (int64_t k = 0; k < n; ++k) {
    const int32_t uu = u[k];
    QREC_REQUIRE(sorted_rowptr[uu + 1] - sorted_rowptr[uu] < num_items,
                 "qrec_sample_pairwise: user %d rated every item", uu);
    uint32_t j = randbelow(st, (uint32_t)num_items);
    while (row_contains(sorted_rowptr, sorted_cols, uu, (int32_t)j)) j = randbelow(st, (uint32_t)num_items);
    out_j[k] = (int32_t)j;
  }
  return QREC_OK;
}

// TBPR's epoch of preference chains (model/ranking/TBPR.py:131-160): for every user of positiveSet (ids in `order`), for
// every positive item i (insertion order) a chain  i > joint > weak > strong > unobserved  of the levels that exist for
// the user -- one choice(list) per non-empty level in that order, then choice(item_list) until the item is not one of the
// user's positives -- emitted as the consecutive (u, a, b) steps of the chain.  Pools: CSR over user ids, items in list
// order.  out_*: capacity 4 * (number of positives of the listed users); out_per_user[k] = steps of order[k].
int qrec_sample_tbpr_epoch(qrec_mt19937* st, int32_t n_order, const int32_t* order, int32_t num_items,
                           const int64_t* pos_rowptr, const int32_t* pos_cols, const int64_t* possorted_rowptr,
                           const int32_t* possorted_cols, const int64_t* joint_rowptr, const int32_t* joint_items,
                           const int64_t* weak_rowptr, const int32_t* weak_items, const int64_t* strong_rowptr,
                           const int32_t* strong_items, int32_t* out_u, int32_t* out_a, int32_t* out_b,
                           int64_t* out_per_user, int64_t* out_n) {
  QREC_REQUIRE(st && pos_rowptr && possorted_rowptr && joint_rowptr && weak_rowptr && strong_rowptr && out_per_user && out_n &&
                   (n_order == 0 || order),
               "qrec_sample_tbpr_epoch: null pointer");
  QREC_REQUIRE(num_items >= 1, "qrec_sample_tbpr_epoch: num_items < 1");
  const int64_t* lrp[3] = {joint_rowptr, weak_rowptr, strong_rowptr};
  const int32_t* lit[3] = {joint_items, weak_items, strong_items};
  int64_t o = 0;
  for (int32_t k = 0; k < n_order; ++k) {
    const int32_t uu = order[k];
    const int64_t start = o;
    QREC_REQUIRE(possorted_rowptr[uu + 1] - possorted_rowptr[uu] < num_items,
                 "qrec_sample_tbpr_epoch: every item is a positive of user %d", uu);
    for (int64_t e = pos_rowptr[uu]; e < pos_rowptr[uu + 1]; ++e) {
      int32_t chain[5];
      int len = 0;
      chain[len++] = pos_cols[e];
      for (int l = 0; l < 3; ++l) {
        const int64_t a = lrp[l][uu], m = lrp[l][uu + 1] - a;
        if (m > 0) chain[len++] = lit[l][a + randbelow(st, (uint32_t)m)];
      }
      uint32_t j = randbelow(st, (uint32_t)num_items);
      while (row_contains(possorted_rowptr, possorted_cols, uu, (int32_t)j)) j = randbelow(st, (uint32_t)num_items);
      chain[len++] = (int32_t)j;
      for (int t = 0; t + 1 < len; ++t) {
        out_u[o] = uu; out_a[o] = chain[t]; out_b[o] = chain[t + 1]; ++o;
      }
    }
    out_per_user[k] = o - start;
  }
  *out_n = o;
  return QREC_OK;
}

// SBPR's minibatch rows (model/ranking/SBPR.py:84-100): per row one social item k = choice(list(FPSet[user].keys()))
// with its friend count S_uk (a user without social feedback draws choice(item_list) and weight 0), then a negative
// j = choice(item_list) until j is neither rated by the user nor in FPSet[user].  choice(seq) = seq[_randbelow(len(seq))];
// item_list is in id order.  fp_items / fp_counts: the users' FPSet in dict (insertion) order; fp_sorted: the same sets
// ascending, for the membership test.
int qrec_sample_sbpr_batch(qrec_mt19937* st, int64_t n, int32_t num_items, const int32_t* u,
                           const int64_t* rated_rowptr, const int32_t* rated_cols, const int64_t* fp_rowptr,
                           const int32_t* fp_items, const int32_t* fp_counts, const int32_t* fp_sorted,
                           int32_t* out_k, int32_t* out_j, int32_t* out_w) {
  QREC_REQUIRE(st && rated_rowptr && fp_rowptr && (n == 0 || (u && out_k && out_j && out_w)),
               "qrec_sample_sbpr_batch: null pointer");
  QREC_REQUIRE(num_items >= 1, "qrec_sample_sbpr_batch: num_items < 1");
  for (int64_t r = 0; r < n; ++r) {
    const int32_t uu = u[r];
    const int64_t f0 = fp_rowptr[uu], nf = fp_rowptr[uu + 1] - f0;
    if (nf == 0) {
      out_k[r] = (int32_t)randbelow(st, (uint32_t)num_items);
      out_w[r] = 0;
    } else {
      QREC_REQUIRE(fp_items && fp_counts && fp_sorted, "qrec_sample_sbpr_batch: null social-feedback arrays");
      const uint32_t t = randbelow(st, (uint32_t)nf);
      out_k[r] = fp_items[f0 + t];
      out_w[r] = fp_counts[f0 + t];
    }
    QREC_REQUIRE((rated_rowptr[uu + 1] - rated_rowptr[uu]) + nf < num_items,
                 "qrec_sample_sbpr_batch: user %d leaves no item to draw a negative from", uu);
    uint32_t j = randbelow(st, (uint32_t)num_items);
    while (row_contains(rated_rowptr, rated_cols, uu, (int32_t)j) || (nf > 0 && row_contains(fp_rowptr, fp_sorted, uu, (int32_t)j)))
      j = randbelow(st, (uint32_t)num_items);
    out_j[r] = (int32_t)j;
  }
  return QREC_OK;
}

int qrec_sample_pointwise(qrec_mt19937* st, int64_t n, int32_t num_items, const int32_t* u,
                          const int32_t* i, const int64_t* sorted_rowptr,
                          const int32_t* sorted_cols, int32_t* out_u, int32_t* out_i,
                          int32_t* out_y) {
  QREC_REQUIRE(st && sorted_rowptr && (n == 0 || (u && i && out_u && out_i && out_y)),
               "qrec_sample_pointwise: null pointer");
  QREC_REQUIRE(num_items >= 1, "qrec_sample_pointwise: num_items < 1");
  int64_t o = 0;
  for (int64_t k = 0; k < n; ++k) {
    const int32_t uu = u[k];
    QREC_REQUIRE(sorted_rowptr[uu + 1] - sorted_rowptr[uu] < num_items,
                 "qrec_sample_pointwise: user %d rated every item", uu);
    out_u[o] = uu; out_i[o] = i[k]; out_y[o] = 1; ++o;
    for (int r = 0; r < 4; ++r) {
      // randint(0, I-1) = 0 + _randbelow(I)
      uint32_t j = randbelow(st, (uint32_t)num_items);
      while (row_contains(sorted_rowptr, sorted_cols, uu, (int32_t)j)) j = randbelow(st, (uint32_t)num_items);
      out_u[o] = uu; out_i[o] = (int32_t)j; out_y[o] = 0; ++o;
    }
  }
  return QREC_OK;
}

int64_t qrec_bpr_order_depth(int64_t n, const int32_t* u, const int32_t* i, const int32_t* j,
                             int32_t num_users, int32_t num_items) {
  if (n <= 0 || !u || !i || !j || num_users <= 0 || num_items <= 0) return 0;
  // level(k) = 1 + max level of the previous toucher of P[u_k], Q[i_k], Q[j_k]
  std::vector<int64_t> lu((size_t)num_users, 0), lq((size_t)num_items, 0);
  int64_t depth = 0;
  for (int64_t k = 0; k < n; ++k) {
    const int32_t uu = u[k], ii = i[k], jj = j[k];
    if (uu < 0 || uu >= num_users || ii < 0 || ii >= num_items || jj < 0 || jj >= num_items) return -1;
    int64_t lv = lu[uu];
    if (lq[ii] > lv) lv = lq[ii];
    if (lq[jj] > lv) lv = lq[jj];
    ++lv;
    lu[uu] = lq[ii] = lq[jj] = lv;
    if (lv > depth) depth = lv;
  }
  return depth;
}

int qrec_bpr_order_prepare(int64_t n, const int32_t* u, const int32_t* i, const int32_t* j,
                           int32_t num_users, int32_t num_items, int32_t* wait_u,
                           int32_t* wait_i, int32_t* wait_j) {
  QREC_REQUIRE(n == 0 || (u && i && j && wait_u && wait_i && wait_j), "qrec_bpr_order_prepare: null pointer");
  QREC_REQUIRE(num_users >= 0 && num_items >= 0, "qrec_bpr_order_prepare: bad sizes");
  std::vector<int32_t> cu((size_t)num_users, 0), cq((size_t)num_items, 0);
  for (int64_t k = 0; k < n; ++k) {
    const int32_t uu = u[k], ii = i[k], jj = j[k];
    QREC_REQUIRE(uu >= 0 && uu < num_users && ii >= 0 && ii < num_items && jj >= 0 && jj < num_items,
                 "qrec_bpr_order_prepare: id out of range at triple %lld", (long long)k);
    QREC_REQUIRE(ii != jj, "qrec_bpr_order_prepare: i == j at triple %lld", (long long)k);
    wait_u[k] = cu[uu]++;
    wait_i[k] = cq[ii]++;
    wait_j[k] = cq[jj]++;
  }
  return QREC_OK;
}

// pointwise streams (u,i): two rows per entry (model/rating/PMF.py:13-22 and siblings)
int64_t qrec_mf_order_depth(int64_t n, const int32_t* u, const int32_t* i, int32_t num_users,
                            int32_t num_items) {
  if (n <= 0 || !u || !i || num_users <= 0 || num_items <= 0) return 0;
  std::vector<int64_t> lu((size_t)num_users, 0), lq((size_t)num_items, 0);
  int64_t depth = 0;
  for (int64_t k = 0; k < n; ++k) {
    const int32_t uu = u[k], ii = i[k];
    if (uu < 0 || uu >= num_users || ii < 0 || ii >= num_items) return -1;
    const int64_t lv = (lu[uu] > lq[ii] ? lu[uu] : lq[ii]) + 1;
    lu[uu] = lq[ii] = lv;
    if (lv > depth) depth = lv;
  }
  return depth;
}

int qrec_mf_order_prepare(int64_t n, const int32_t* u, const int32_t* i, int32_t num_users,
                          int32_t num_items, int32_t* wait_u, int32_t* wait_i) {
  QREC_REQUIRE(n == 0 || (u && i && wait_u && wait_i), "qrec_mf_order_prepare: null pointer");
  QREC_REQUIRE(num_users >= 0 && num_items >= 0, "qrec_mf_order_prepare: bad sizes");
  std::vector<int32_t> cu((size_t)num_users, 0), cq((size_t)num_items, 0);
  for (int64_t k = 0; k < n; ++k) {
    const int32_t uu = u[k], ii = i[k];
    QREC_REQUIRE(uu >= 0 && uu < num_users && ii >= 0 && ii < num_items,
                 "qrec_mf_order_prepare: id out of range at entry %lld", (long long)k);
    wait_u[k] = cu[uu]++;
    wait_i[k] = cq[ii]++;
  }
  return QREC_OK;
}

// RSTE's rating pass (model/rating/RSTE.py:20-64): entry (u, i) reads P[u], Q[i] and the followee rows P[f]
// (f_rowptr / f_cols, a CSR over users) and writes P[u], Q[i].  One pass, O(n + sum of the entries' out-degrees).
int qrec_rste_order_prepare(int64_t n, const int32_t* u, const int32_t* i, int32_t num_users, int32_t num_items,
                            const int64_t* f_rowptr, const int32_t* f_cols, int32_t* wait_u, int32_t* wait_i,
                            int32_t* wait_reads_u, int64_t* pos_rowptr, int32_t* pos, int64_t* depth) {
  QREC_REQUIRE(num_users >= 0 && num_items >= 0, "qrec_rste_order_prepare: bad sizes");
  QREC_REQUIRE(n >= 0 && n < (int64_t(1) << 31), "qrec_rste_order_prepare: n=%lld outside [0, 2^31)", (long long)n);
  QREC_REQUIRE(f_rowptr && pos_rowptr && depth, "qrec_rste_order_prepare: null pointer");
  QREC_REQUIRE(n == 0 || (u && i && wait_u && wait_i && wait_reads_u && pos), "qrec_rste_order_prepare: null pointer");
  QREC_REQUIRE(f_rowptr[0] == 0, "qrec_rste_order_prepare: followee rowptr must start at 0");
  for (int32_t r = 0; r < num_users; ++r)
    QREC_REQUIRE(f_rowptr[r + 1] >= f_rowptr[r], "qrec_rste_order_prepare: followee rowptr falls at user %d", r);
  const int64_t nnz = f_rowptr[num_users];
  QREC_REQUIRE(nnz == 0 || f_cols, "qrec_rste_order_prepare: null followee list");
  for (int64_t j = 0; j < nnz; ++j)
    QREC_REQUIRE(f_cols[j] >= 0 && f_cols[j] < num_users, "qrec_rste_order_prepare: followee %lld out of range",
                 (long long)j);
  for (int64_t k = 0; k < n; ++k)
    QREC_REQUIRE(u[k] >= 0 && u[k] < num_users && i[k] >= 0 && i[k] < num_items,
                 "qrec_rste_order_prepare: id out of range at entry %lld", (long long)k);
  // writes / foreign reads counted so far, and the dependency level of the last write / latest read of each row
  std::vector<int32_t> cu((size_t)num_users, 0), cq((size_t)num_items, 0), cr((size_t)num_users, 0);
  std::vector<int64_t> lw((size_t)num_users, 0), lr((size_t)num_users, 0), lq((size_t)num_items, 0);
  int64_t deep = 0;
  for (int64_t k = 0; k < n; ++k) {
    const int32_t uu = u[k], ii = i[k];
    wait_u[k] = cu[uu]++;
    wait_i[k] = cq[ii]++;
    wait_reads_u[k] = cr[uu];
    int64_t lv = lw[uu] > lr[uu] ? lw[uu] : lr[uu];
    if (lq[ii] > lv) lv = lq[ii];
    for (int64_t j = f_rowptr[uu]; j < f_rowptr[uu + 1]; ++j)
      if (f_cols[j] != uu && lw[f_cols[j]] > lv) lv = lw[f_cols[j]];
    ++lv;
    for (int64_t j = f_rowptr[uu]; j < f_rowptr[uu + 1]; ++j) {
      const int32_t f = f_cols[j];
      if (f == uu) continue;
      ++cr[f];
      if (lv > lr[f]) lr[f] = lv;
    }
    lw[uu] = lq[ii] = lv;
    if (lv > deep) deep = lv;
  }
  *depth = deep;
  // entry positions by user, ascending: rows of the CSR are the users' write counts (cu)
  pos_rowptr[0] = 0;
  for (int32_t r = 0; r < num_users; ++r) pos_rowptr[r + 1] = pos_rowptr[r] + cu[r];
  std::vector<int64_t> fill(pos_rowptr, pos_rowptr + num_users);
  for (int64_t k = 0; k < n; ++k) pos[fill[u[k]]++] = (int32_t)k;
  return QREC_OK;
}

// The trust-neighbourhood user pass (K17, social_pass_kernels.cu) over the visiting order visit[0..n): pos[u] = the
// position of user u in it, -1 when u is not visited; *depth = the longest chain of users each waiting for an earlier
// followee or follower (f_* / g_*: the followee and follower CSRs over users, with f_nnz / g_nnz columns).
int qrec_social_order_prepare(int64_t n, const int32_t* visit, int32_t num_users, const int64_t* f_rowptr,
                              const int32_t* f_cols, int64_t f_nnz, const int64_t* g_rowptr, const int32_t* g_cols,
                              int64_t g_nnz, int32_t* pos, int64_t* depth) {
  QREC_REQUIRE(num_users >= 0 && n >= 0 && n <= num_users, "qrec_social_order_prepare: n=%lld, num_users=%d",
               (long long)n, num_users);
  QREC_REQUIRE(f_rowptr && g_rowptr && depth && (num_users == 0 || pos) && (n == 0 || visit),
               "qrec_social_order_prepare: null pointer");
  const int64_t* rowptrs[2] = {f_rowptr, g_rowptr};
  const int32_t* colss[2] = {f_cols, g_cols};
  const int64_t nnzs[2] = {f_nnz, g_nnz};
  for (int t = 0; t < 2; ++t) {
    const int64_t* rp = rowptrs[t];
    QREC_REQUIRE(rp[0] == 0 && rp[num_users] == nnzs[t],
                 "qrec_social_order_prepare: %s rowptr must run from 0 to %lld", t ? "follower" : "followee",
                 (long long)nnzs[t]);
    for (int32_t r = 0; r < num_users; ++r)
      QREC_REQUIRE(rp[r + 1] >= rp[r], "qrec_social_order_prepare: %s rowptr falls at user %d",
                   t ? "follower" : "followee", r);
    QREC_REQUIRE(nnzs[t] == 0 || colss[t], "qrec_social_order_prepare: null column list");
    for (int64_t j = 0; j < nnzs[t]; ++j)
      QREC_REQUIRE(colss[t][j] >= 0 && colss[t][j] < num_users, "qrec_social_order_prepare: %s %lld out of range",
                   t ? "follower" : "followee", (long long)j);
  }
  for (int32_t r = 0; r < num_users; ++r) pos[r] = -1;
  for (int64_t k = 0; k < n; ++k) {
    const int32_t uu = visit[k];
    QREC_REQUIRE(uu >= 0 && uu < num_users, "qrec_social_order_prepare: visit %lld out of range", (long long)k);
    QREC_REQUIRE(pos[uu] < 0, "qrec_social_order_prepare: user %d visited twice", uu);
    pos[uu] = (int32_t)k;
  }
  std::vector<int64_t> level((size_t)num_users, 0);
  int64_t deep = 0;
  for (int64_t k = 0; k < n; ++k) {
    const int32_t uu = visit[k];
    int64_t lv = 0;
    for (int t = 0; t < 2; ++t)
      for (int64_t j = rowptrs[t][uu]; j < rowptrs[t][uu + 1]; ++j) {
        const int32_t v = colss[t][j];
        if (v != uu && pos[v] >= 0 && pos[v] < k && level[v] > lv) lv = level[v];
      }
    level[uu] = ++lv;
    if (lv > deep) deep = lv;
  }
  *depth = deep;
  return QREC_OK;
}

}  // extern "C"
