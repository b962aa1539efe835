"""Where the tolerance of tests/test_cli_gpu.py's training comparison comes from.

fp32 training sums some gradients with atomics, so repeated runs of the same loop are not always bit-identical, and Adam
carries a last-bit difference into the weights.  For each case of that test this runs the train command's loop in-process
`--runs` times and prints the weight distances (tests/test_cli_gpu.py::weight_distance) between repeated runs, next to
the distances a wrong data seed, initialisation seed, dropout seed, learning rate, rate decay or iteration count makes.

    python tools/measure_train_spread.py [--runs 10]"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import test_cli_gpu as T  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    a = ap.parse_args()
    n = 2 * T.SPLITS["train"]                                       # the test's 2 epochs of batchSize 1
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for enc, dec in T.CASES:
            os.makedirs(os.path.join(d, enc))
            _, fo = T.write_files(os.path.join(d, enc), enc, dec)
            p = dict(T._params(enc, dec), batchSize=1)
            runs = [T.train_inproc(p, fo, n)[0] for _ in range(a.runs)]
            pairs = [T.weight_distance(x, y) for i, x in enumerate(runs) for y in runs[i + 1:]]
            wrong = {
                "data seed 1235": T.train_inproc(p, fo, n, data_seed=1235)[0],
                "init seed 1235": T.train_inproc(p, fo, n, init_seed=1235)[0],
                "dropout seed 1235": T.train_inproc(dict(p, seed=1235), fo, n)[0],
                "learningRate x1.01": T.train_inproc(dict(p, learningRate=1.01e-3), fo, n)[0],
                "no rate decay": T.train_inproc(dict(p, lrDecayRate=1.0), fo, n)[0],
                "one iteration less": T.train_inproc(p, fo, n - 1)[0],
            }
            out["%s+%s" % (enc, dec)] = {
                "repeated runs": {"pairs": len(pairs), "identical_pairs": sum(x["max"] == 0.0 for x in pairs),
                                  "max": max(x["max"] for x in pairs), "frac_1e-5": max(x["frac_1e-5"] for x in pairs)},
                "wrong": {k: min((T.weight_distance(w, r) for r in runs), key=lambda x: x["frac_1e-5"])
                          for k, w in wrong.items()}}
            print(json.dumps({"%s+%s" % (enc, dec): out["%s+%s" % (enc, dec)]}), flush=True)


if __name__ == "__main__":
    main()
