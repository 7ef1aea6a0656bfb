#!/usr/bin/env python
"""Mint golden vectors at embedding widths 32, 96 and 192 from the UNMODIFIED reference (a checkout of HKUDS/MMSSL named by
$MMSSL_REFERENCE), run on CPU.  Same recipe and same short run as make_golden.py; the only difference is the reference's own
`--embed_size` flag (and, for the d = 192 case, `--head_num 1`), appended to the command line its modules parse at import time.
The d = 192 case is small (32 users, 24 items, one attention head) so that its file stays near the size of the other golden
files: its [head_num * d, d] attention weight and gradient, and the d x d weights, alone are ~0.7 MB at one head.

    python tests/golden/make_golden_width.py            # writes tests/golden/width_d*.npz
"""
import argparse
import importlib
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden  # noqa: E402

CASES = {
    # name: (embed_size, extra reference flags, and make_golden's case fields)
    "width_d32_train_rand_k3": dict(d=32, U=203, I=150, dv=72, dt=24, B=96, ws="[32,32,32]", modal="random", train=True, seed=7),
    "width_d96_train_empty_k2": dict(d=96, U=180, I=97, dv=40, dt=56, B=50, ws="[96,96]", modal="empty", train=True, seed=11),
    "width_d192_eval_alias_k2": dict(d=192, flags=["--head_num", "1"], U=32, I=24, dv=24, dt=16, B=16, ws="[192,192]", modal="alias",
                                     train=False, seed=2022),
}


def run_case(name):
    c = dict(CASES[name])
    d = c.pop("d")
    flags = c.pop("flags", [])
    make_golden.CASES[name] = c
    real_import = importlib.import_module

    def import_module(mod, *a, **k):
        if mod == "main":       # make_golden.run_case has just set sys.argv for the reference's parser
            sys.argv += ["--embed_size", str(d)] + flags
        return real_import(mod, *a, **k)

    importlib.import_module = import_module
    make_golden.run_case(name)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    a, _ = ap.parse_known_args()
    if a.case:
        run_case(a.case)
    else:
        for n in CASES:
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--case", n])
