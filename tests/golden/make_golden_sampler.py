#!/usr/bin/env python
"""Records what the UNMODIFIED reference sampler (utility/load_data.py:Data.sample, :153-191) draws on
tests/golden/dataset_small for fixed seeds of `random` and `numpy.random` -> tests/golden/sampler_small.json.
Runs only where the reference checkout ($MMSSL_REFERENCE) exists."""
import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF  # noqa: E402


def main():
    d = os.path.join(HERE, "dataset_small")
    sys.path.insert(0, REF)
    os.chdir(REF)
    sys.argv = ["x", "--debug"]
    from utility.load_data import Data
    out = {}
    for batch in (16, 80):                 # 80 > n_users: the with-replacement branch (load_data.py:156-157)
        dg = Data(path=d, batch_size=batch)
        random.seed(11)
        np.random.seed(11)
        out[str(batch)] = [[[int(v) for v in part] for part in dg.sample()] for _ in range(3)]
    json.dump(out, open(os.path.join(HERE, "sampler_small.json"), "w"))
    print("wrote sampler_small.json", {k: len(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
