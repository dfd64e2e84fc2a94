"""TEST INFRASTRUCTURE: a short NumPy restatement of the reference's clustered fairness metrics over recommendation
dicts, written from their definitions (BiasDisparity: arXiv 1811.01461; MAD; REO / RSP), independent of
elliot_b200/fairness.py.  evaluate() gives {result key: value} in the reference's key order for one split at cutoff k."""
import warnings

import numpy as np
import pandas as pd


def _clusters(path):
    if not path:
        return {}, 1
    df = pd.read_csv(path, sep="\t", header=None)
    return dict(zip(df[0].tolist(), df[1].tolist())), int(df[1].nunique())


def _mad(values_by_cluster, n):
    avg = [np.mean(v) if v else np.nan for v in (values_by_cluster.get(c, []) for c in range(n))]
    diffs = [abs(avg[i] - avg[j]) for i in range(n) for j in range(i + 1, n)]
    return float(np.mean(diffs)) if diffs else float("nan")


def evaluate(data, recs, split, k, entries, thr=None):
    thr = data.config.evaluation.relevance_threshold if thr is None else thr
    recs = {u: r[:k] for u, r in recs.items() if split.get(u)}
    rel = {u: {i: 2.0 ** (s - thr + 1) - 1 for i, s in split[u].items() if s >= thr} for u in recs}
    train = data.train_dict
    out = {}
    with warnings.catch_warnings(), np.errstate(divide="ignore", invalid="ignore"):
        warnings.simplefilter("ignore")
        for e in entries:
            m = e["metric"]
            if m.startswith("UserMAD"):
                cl, n = _clusters(e.get("clustering_file"))
                per = {}
                for u, r in recs.items():
                    if rel[u] and u in cl:
                        if m == "UserMADrating":
                            v = np.mean([s for _, s in r]) if r else np.nan
                        else:
                            ideal = sorted(rel[u].values(), reverse=True)[:k]
                            idcg = sum(g / np.log2(j + 2) for j, g in enumerate(ideal))
                            dcg = sum(rel[u].get(i, 0) / np.log2(j + 2) for j, (i, _) in enumerate(r))
                            v = dcg / idcg if dcg > 0 else 0.0
                        per.setdefault(cl[u], []).append(v)
                out[f"{m}_{e.get('clustering_name', '')}"] = _mad(per, n)
            elif m.startswith("ItemMAD"):
                cl, n = _clusters(e.get("clustering_file"))
                cnt, tot = {}, {}
                for u, r in recs.items():
                    if rel[u]:
                        for i, s in r:
                            cnt[i] = cnt.get(i, 0) + 1
                            add = rel[u].get(i, 0) if m == "ItemMADranking" else (s if i in rel[u] else 0)
                            tot[i] = tot.get(i, 0) + add
                per = {}
                for i in cnt:
                    if i in cl:
                        per.setdefault(cl[i], []).append(tot[i] / cnt[i])
                out[f"{m}_{e.get('clustering_name', '')}"] = _mad(per, n)
            elif m in ("REO", "RSP"):
                cl, n = _clusters(e.get("clustering_file"))
                name = e.get("clustering_name", "") if e.get("clustering_file") else ""
                members = {c: {i for i, cc in cl.items() if cc == c} for c in range(n)} if cl else {}
                num, den = np.zeros(n), np.zeros(n)
                for u, r in recs.items():
                    if m == "REO" and not rel[u]:
                        continue
                    listed = {i for i, _ in r}
                    if m == "REO":
                        listed &= set(rel[u])
                    for c, mem in members.items():
                        num[c] += len(listed & mem)
                        den[c] += len((mem & set(rel[u]) if m == "REO" else mem) - set(train[u]))
                pr = num / den
                out.update({f"{m}-ProbToBeRanked_items:{name}-{c}": float(pr[c]) for c in range(n)})
                out[f"{m}_items:{name}"] = float(np.std(pr) / np.mean(pr))
            else:
                ucl, nu = _clusters(e.get("user_clustering_file"))
                icl, ni = _clusters(e.get("item_clustering_file"))
                un = e.get("user_clustering_name", "") if ucl else ""
                iname = e.get("item_clustering_name", "") if icl else ""
                pc = np.array([sum(1 for v in icl.values() if v == c) / len(icl) for c in range(ni)]) if icl else np.ones(1)

                def bias(lists):
                    cat = np.zeros((nu, ni))
                    for u, items in lists.items():
                        g = ucl.get(u) if ucl else 0
                        for i in items:
                            c = icl.get(i) if icl else 0
                            if g is not None and c is not None:
                                cat[g, c] += 1
                    return cat / cat.sum(1, keepdims=True) / pc
                br = bias({u: [i for i, _ in r] for u, r in recs.items()})
                bs = bias({u: list(t) for u, t in train.items()})
                val = {"BiasDisparityBR": br, "BiasDisparityBS": bs, "BiasDisparityBD": (br - bs) / bs}[m]
                out.update({f"{m}_users:{un}-{g}_items:{iname}-{c}": float(val[g, c]) for g in range(nu) for c in range(ni)})
    return out
