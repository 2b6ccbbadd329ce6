"""Generate tests/golden/lr_schedule_pins.json by RUNNING THE REFERENCE'S OWN LR SCHEDULE
(training/util/lr_scheduler.py `IterExponential`, imported by path from a read-only checkout of
VisualComputingInstitute/diffusion-e2e-ft) at the iteration counts the recipes reach: both scripts build
`IterExponential(lr_total_iter_length * N, 0.01, warmup * N)` with 20000 optimizer steps and 100 warm-up steps
(training/train.py:355-357, GeoWizard train_depth_normal.py:468-471), N = accelerate's num_processes.  The values are
stored with full float64 precision, so tests/test_training_state_cpu.py compares `training.IterExponential` with them
exactly and needs no reference checkout.

    python tests/golden/make_lr_schedule_pins.py <path to the reference checkout>
"""
import importlib.util
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIGS = [(20000, 0.01, 100, 1), (20000, 0.01, 100, 2), (20000, 0.01, 100, 8), (300, 0.05, 0, 1), (50, 0.01, 10, 1)]


def main(ref):
    spec = importlib.util.spec_from_file_location("ref_lr_scheduler", os.path.join(ref, "training/util/lr_scheduler.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    pins = []
    for total, final, warmup, n in CONFIGS:
        fn = mod.IterExponential(total_iter_length=total * n, final_ratio=final, warmup_steps=warmup * n)
        iters = sorted(set(list(range(0, 260 * n)) + [k * n for k in range(0, total + 50, 97)] +
                           [total * n - 1, total * n, total * n + 1, warmup * n, max(0, warmup * n - 1)]))
        pins.append(dict(total_iter_length=total * n, final_ratio=final, warmup_steps=warmup * n,
                         n_iter=iters, value=[float(fn(i)) for i in iters],
                         attributes={k: v for k, v in vars(fn).items()}))
    with open(os.path.join(HERE, "lr_schedule_pins.json"), "w") as f:
        json.dump(pins, f, separators=(",", ":"))


if __name__ == "__main__":
    main(sys.argv[1])
