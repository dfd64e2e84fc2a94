#!/usr/bin/env python
"""MostPop and Random phase timings on one GPU; prints one JSON line per data set and a summary line.

For each data set the lists of every user at k = 10 are built once to warm up and then --repeat times, each phase timed
through the models' marks (tools/benchlib.py), medians reported: MostPop's popularity (integer atomics over the train
CSR), order (one stable sort of n_items keys) and lists (one warp per user); Random's stream (the serial one-warp walk
of the MT19937 words in user order, with the generation of the words it reads and one host synchronise per buffer) and
select (the r-th item outside each train row).  The card's name, power limit and SM clock are read in the same run.

Data sets (benchlib): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706); ML-20M-shaped = 138 493 x
26 744, ~18.4 M ratings.

    python tools/unpersonalized_bench.py [--repeat N] [--skip-ml20m]
"""
import argparse
import json

import benchlib as bl
from elliot_b200.recommender.unpersonalized import MostPopLists, RandomLists


def run(name, u, i, r, U, I, repeat):
    data = bl.Data(u, i, r, U, I)
    mp, rd = MostPopLists(data, bl.DEV), RandomLists(data, 42, bl.DEV)

    def mostpop(mark):
        mp.initialize(mark)
        mp.topk(10, mark=mark)
    t_mp = bl.repeat(mostpop, repeat)
    t_rd = bl.repeat(lambda mark: rd.topk(10, mark=mark), repeat)
    words = rd.stream.consumed / (repeat + 1)
    row = {"data": name, "users": U, "items": I, "nnz": int(len(u)),
           "MostPop_ms": {k: round(v, 3) for k, v in t_mp.items()},
           "Random_ms": {k: round(v, 3) for k, v in t_rd.items()},
           "Random_words_per_call": round(words), "Random_stream_ns_per_word": round(t_rd["stream"] * 1e6 / words, 2)}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--skip-ml20m", action="store_true")
    args = ap.parse_args()
    res = bl.card()
    rows = [run("C1", *bl.c1_matrix(), args.repeat)]
    if not args.skip_ml20m:
        rows.append(run("ML-20M-shape", *bl.ml20m_matrix(), args.repeat))
    res["runs"] = rows
    res["sm_clock_mhz_after"] = bl.card()["sm_clock_mhz"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
