"""Float64 restatement of the reference's memory-based rating models (model/rating/UserKNN.py, ItemKNN.py,
SlopeOne.py with util/qmath.py), kept to the operation order that decides their bits:

  * similarities sum over x1's keys in insertion order, restricted to x2's, with CPython's `** 2` for the squares
    (glibc pow, not numpy's square);
  * the candidate list of the query at position p is every earlier query (cold ones included) with the similarity
    the earlier query computed -- similarity(earlier row, this row) -- then every other training row in id order with
    similarity(this row, it); a cold query lists every training row with similarity 0.  The list is sorted by
    similarity descending, stably (the reference's SymmetricMatrix insertion order under sorted(..., reverse=True));
  * rows sharing no key have similarity 0 without any arithmetic, so only rows found through the columns are computed.

Rows are dicts {column name: value} in insertion order (Rating.trainSet_u / trainSet_i).  Test infrastructure: the
engine never imports this module.
"""
from collections import defaultdict
from math import sqrt


def similarity(x1, x2, sim):
    """util/qmath.py: similarity -- pearson_sp, euclidean_sp, or cosine_sp for any other name."""
    if sim == 'pcc':
        total = d1 = d2 = 0
        overlapped = False
        if not x1 or not x2:
            return 0
        m1 = sum(x1.values()) / len(x1)
        m2 = sum(x2.values()) / len(x2)
        for k in x1:
            if k in x2:
                total += (x1[k] - m1) * (x2[k] - m2)
                d1 += (x1[k] - m1) ** 2
                d2 += (x2[k] - m2) ** 2
                overlapped = True
        den = sqrt(d1) * sqrt(d2)
        if den == 0:
            return 1 if overlapped else 0
        return total / den
    if sim == 'euclidean':
        total = 0
        for k in x1:
            if k in x2:
                total += x1[k] ** 2 - x2[k] ** 2
        return 0 if total == 0 else 1 / total
    total = d1 = d2 = 0
    for k in x1:
        if k in x2:
            total += x1[k] * x2[k]
            d1 += x1[k] ** 2
            d2 += x2[k] ** 2
    den = sqrt(d1) * sqrt(d2)
    return 0 if den == 0 else total / den


def _columns(rows):
    by_col = defaultdict(list)
    for name, row in rows.items():
        for c in row:
            by_col[c].append(name)
    return by_col


def sorted_lists(rows, train_names, queries, sim, keep=None):
    """{query: [(name, sim), ...]}: each query's candidate list sorted as the reference sorts it (first `keep`
    entries when keep is not None).  rows: the training rows by name; train_names: the training rows in id order;
    queries: the query list (testSet_u / testSet_i order)."""
    by_col = _columns(rows)
    out = {}
    done = []
    for q in queries:
        if q not in rows:
            lst = [(v, 0) for v in train_names]
        else:
            xq = rows[q]
            sharing = {v for c in xq for v in by_col[c] if v != q}
            earlier = set(done)
            lst = [(e, similarity(rows[e], xq, sim) if e in sharing else 0) for e in done]
            lst += [(v, similarity(xq, rows[v], sim) if v in sharing else 0) for v in train_names
                    if v != q and v not in earlier]
        lst.sort(key=lambda d: d[1], reverse=True)
        out[q] = lst if keep is None else lst[:keep]
        done.append(q)
    return out


def knn_predict(top, k, q, probe_rows, probe, query_mean, neighbour_means, global_mean, minus_one_unrated):
    """UserKNN / ItemKNN predictForRating: q's first min(k, len) neighbours n with `probe` in probe_rows[n] (the
    neighbour's training row; UserKNN also skips a stored -1) add sim*(r - mean[n]) and sim.  query_mean is None for a
    query with no training row.  Raises ZeroDivisionError as the reference does."""
    s, denom = 0, 0
    for name, w in top[q][:max(min(k, len(top[q])), 0)]:
        row = probe_rows.get(name)
        if row is None or probe not in row:
            continue
        r = row[probe]
        if minus_one_unrated and r == -1:
            continue
        s += w * (r - neighbour_means[name])
        denom += w
    if s == 0:
        return global_mean if query_mean is None else query_mean
    return (query_mean if query_mean is not None else global_mean) + s / float(denom)


def slopeone_tables(items, train_items, test_items):
    """SlopeOne.computeAverage: {test item: ({item: diff average}, {item: count})} against every training item."""
    diff_avg, freq = {}, {}
    by_user = defaultdict(dict)
    for j in train_items:
        for u, r in items[j].items():
            by_user[u][j] = r
    for i in test_items:
        x1 = items.get(i, {})
        acc = {}
        for u in x1:
            for j, b in by_user[u].items():
                d, n = acc.get(j, (0.0, 0))
                acc[j] = (d + (x1[u] - b), n + 1)
        diff_avg[i] = {j: (acc[j][0] / acc[j][1] if j in acc else 0) for j in train_items}
        freq[i] = {j: (acc[j][1] if j in acc else 0) for j in train_items}
    return diff_avg, freq


def slopeone_predict(diff_avg, freq, user_rows, user_means, item_means, global_mean, u, i):
    """SlopeOne.predictForRating."""
    if u in user_rows:
        s, fs = 0, 0
        for j, r in user_rows[u].items():
            s += (r + diff_avg[i][j]) * freq[i][j]
            fs += freq[i][j]
        return user_means[u] if fs == 0 else float(s) / fs
    if i in item_means:
        return item_means[i]
    return global_mean
