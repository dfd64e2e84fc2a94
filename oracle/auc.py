"""The reference's AUC and GAUC (elliot/evaluation/metrics/accuracy/AUC/auc.py, gauc.py) restated over explicit full
recommendation lists, and the per-user counts the device rank pass (eb_score_rank_*) produces, read off those lists.

A full list is every item the model ranks for the user, in list order.  For a user u with relevant items R_u (binary
relevance of the split, test-only items included), train profile size |train_u| and the i-th positive found at list
position r_i, the reference's term is (neg_u - r_i + i) / neg_u with neg_u = num_items - |train_u| - |R_u| + 1.  AUC
averages every term of every user with |R_u| > 0 (np.average of the flattened list: NaN when there is none); GAUC
averages sum(terms) / |R_u| over those users.  Python int / int division: neg_u = 0 with a positive raises
ZeroDivisionError, as in the reference."""
import warnings

import numpy as np


def user_terms(full_list, rel, num_items, train_size):
    neg = num_items - train_size - len(rel) + 1
    rel = set(rel)
    pos = [r for r, i in enumerate(full_list) if i in rel]
    return [(neg - r + p) / neg for p, r in enumerate(pos)]


def auc_gauc(lists, rels, num_items, train_sizes):
    """(AUC, GAUC) of {user: full list}, {user: relevant items} and {user: |train_u|}; users without relevant items are
    skipped."""
    users = [u for u in lists if len(rels.get(u, []))]
    terms = [user_terms(lists[u], rels[u], num_items, train_sizes[u]) for u in users]
    with warnings.catch_warnings():                                 # np.average([]) warns and gives NaN
        warnings.simplefilter("ignore", RuntimeWarning)
        auc = float(np.average([t for ts in terms for t in ts]))
        gauc = float(np.average([sum(ts) / len(rels[u]) for u, ts in zip(users, terms)]))
    return auc, gauc


def rank_counts(full_list, rel):
    """(n_pos, sum_c, c) of one user: the positives found in the list, the sum over them of the non-relevant entries
    ahead of each, and those counts in list order."""
    rel = set(rel)
    c, ahead = [], 0
    for i in full_list:
        if i in rel:
            c.append(ahead)
        else:
            ahead += 1
    return len(c), int(sum(c)), c
