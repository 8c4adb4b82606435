"""Compare two `bench.py --dump-outputs` directories (for example the same run with two builds of the library).

    python scripts/compare_dumps.py DIR_A DIR_B [--grad-rtol 1e-5]

Everything the forward pass computes (losses, scores, the logits sample) must be bit-identical; gradients may differ by the
summation order of the fp32 weight-gradient atomics, so `grads_norm` is held to a relative tolerance and the gradient sample
is reported. Exit status 0 when both hold."""
import argparse
import os
import sys

import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("a")
    ap.add_argument("b")
    ap.add_argument("--grad-rtol", type=float, default=1e-5)
    args = ap.parse_args()
    names = sorted(f[:-4] for f in os.listdir(args.a) if f.endswith(".npy"))
    missing = sorted(set(f[:-4] for f in os.listdir(args.b) if f.endswith(".npy")) ^ set(names))
    ok = not missing
    if missing:
        print(f"entries present in only one dump: {missing}")
    for n in names:
        if n in missing:
            continue
        x = np.load(os.path.join(args.a, n + ".npy"))
        y = np.load(os.path.join(args.b, n + ".npy"))
        if n.startswith("grads"):
            if n == "grads_norm":
                rel = abs(float(x) - float(y)) / max(abs(float(x)), 1e-30)
                good = rel <= args.grad_rtol
                print(f"{n}: {float(x):.9g} vs {float(y):.9g}, relative difference {rel:.3e} {'OK' if good else 'FAIL'}")
                ok &= good
            elif n == "grads_sample":
                d = np.abs(x.astype(np.float64) - y)
                scale = np.abs(x).max()
                print(f"{n}: max |diff| {d.max():.3e} of max |value| {scale:.3e}, {np.count_nonzero(d)} of {d.size} entries differ")
            else:
                same = np.array_equal(x, y)
                print(f"{n}: {'identical' if same else 'DIFFERENT'}")
                ok &= same
            continue
        same = x.shape == y.shape and np.array_equal(x, y, equal_nan=True)
        print(f"{n}: {'bit-identical' if same else 'DIFFERENT'} {tuple(np.shape(x))}")
        ok &= same
    print("COMPARE", "OK" if ok else "FAIL")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
