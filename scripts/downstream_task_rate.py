"""Cost of the downstream-task score: CUDA-event time of `dv_downstream_logistic_cv` for each training size at the
dSprites shape (D = 10; factors of 3, 6, 40, 32 and 32 values; 5,000 test rows) and, with --limits, at the limits
(D = 128, a 256-value factor, 32,768 training rows); the whole `downstream_task` for each predictor; the largest
Newton step count per C; the workspace bytes; and sklearn's host time for the same logistic fits
(LogisticRegressionCV(Cs=10, cv=KFold(5)) at its defaults) up to --sklearn-max rows.  Prints the card and its power
limit first.  Writes nothing."""
import argparse
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "disentangling-vae_b200"))

from disvae import _native as N  # noqa: E402
from disvae import evaluate  # noqa: E402

DEV = torch.device("cuda", 0)


def code(lat, D, seed, noise=0.2):
    """Latent d follows factor d (scaled to [0, 1)) plus noise; the latents past the factors are noise."""
    g = torch.Generator().manual_seed(seed)
    v = torch.from_numpy(np.stack(np.unravel_index(np.arange(int(np.prod(lat))), lat), 1)).float()
    x = torch.randn(v.size(0), D, generator=g)
    K = min(D, len(lat))
    x[:, :K] = v[:, :K] / torch.tensor(lat[:K]).float() + noise * x[:, :K]
    return x.to(DEV)


def timed(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times)), out


def kernel_rows(x, lat, sizes, num_test, reps, label):
    gen = torch.Generator(device=DEV)
    gen.manual_seed(0)
    for size in sizes:
        tr = torch.randint(x.shape[0], (size,), generator=gen, device=DEV)
        te = torch.randint(x.shape[0], (num_test,), generator=gen, device=DEV)
        _, train_cls, _, n_classes, counts, _ = evaluate.sap_labels(lat, tr, te)
        K, S = counts.shape
        ms, out = timed(lambda: evaluate.downstream_logistic_cv(x, tr, te, train_cls, n_classes, S), reps)
        iters = out[4].cpu()
        folds = iters[:, :-1].view(K, 5, -1)
        per_c = folds.max(1)[0].max(0)[0].tolist()
        nbytes = N.lib().dv_downstream_workspace_bytes(x.shape[1], size, K, S, 10)
        print("%s n=%5d: dv_downstream_logistic_cv %9.1f ms  workspace %7.1f MB  largest Newton steps per C %s, "
              "refit %d, non-converged %d" % (label, size, ms, nbytes / 2 ** 20, per_c, int(iters[:, -1].max()),
                                             int((iters < 0).sum())))


def sklearn_rows(x, lat, sizes, num_test):
    from sklearn.linear_model import LogisticRegressionCV
    from sklearn.model_selection import KFold
    gen = torch.Generator(device=DEV)
    gen.manual_seed(0)
    mu = x.cpu().numpy()
    for size in sizes:
        tr = torch.randint(x.shape[0], (size,), generator=gen, device=DEV)
        te = torch.randint(x.shape[0], (num_test,), generator=gen, device=DEV)
        _, train_cls, _, _, _, _ = evaluate.sap_labels(lat, tr, te)
        xt, cls = mu[tr.cpu().numpy()], train_cls.cpu().numpy()
        t0 = time.perf_counter()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for k in range(len(cls)):
                if len(np.unique(cls[k])) > 1:
                    LogisticRegressionCV(Cs=10, cv=KFold(n_splits=5)).fit(xt, cls[k])
        print("sklearn n=%5d: LogisticRegressionCV fits of every factor on the host: %.2f s"
              % (size, time.perf_counter() - t0))


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--limits", action="store_true")
    ap.add_argument("--sklearn-max", type=int, default=1000)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    lat = [1, 3, 6, 40, 32, 32]
    x = code(lat[1:], 10, 1)
    sizes = (10, 100, 1000, 10000)
    kernel_rows(x, lat, sizes, 5000, a.reps, "dSprites")
    for predictor in evaluate.DOWNSTREAM_PREDICTORS:
        ms, _ = timed(lambda: evaluate.downstream_task(x, lat, predictor=predictor, seed=0), 1)
        print("downstream_task(%s), sizes %s, 5000 test rows: %.1f ms" % (predictor, sizes, ms))
    if a.limits:
        lat_l = [256, 2, 64]
        kernel_rows(code(lat_l, 128, 2), lat_l, (32768,), 5000, 1, "limits")
    sklearn_rows(x, lat, [s for s in sizes if s <= a.sklearn_max], 5000)


if __name__ == "__main__":
    main()
