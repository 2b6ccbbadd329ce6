"""Run the kernel parity checks on the GPU and save a table to out/kernel_checks.json.

Checks run sequentially inside a worker process; when one poisons the CUDA context (trap / illegal
address) or hangs, the worker is abandoned and a fresh one continues with the remaining checks, so
one broken kernel cannot hide the others.
    python tools/gpu_kernel_check.py [name ...]
"""
import json
import os
import subprocess
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def worker(names):
    import torch
    from kernel_checks import CHECKS
    for n in names:
        try:
            err, tol = CHECKS[n]()
            torch.cuda.synchronize()
            print("RESULT", json.dumps({"name": n, "err": err, "tol": tol}), flush=True)
        except Exception as e:  # noqa: BLE001
            msg = "".join(traceback.format_exception_only(type(e), e))[-500:]
            print("RESULT", json.dumps({"name": n, "error": msg}), flush=True)
            if "CUDA" in msg or "cuda" in msg or "launch" in msg:
                return


if len(sys.argv) > 1 and sys.argv[1] == "--worker":
    worker(sys.argv[2:])
    sys.exit(0)

from kernel_checks import CHECKS  # noqa: E402

todo = sys.argv[1:] or list(CHECKS)
results = {}
while todo:
    try:
        r = subprocess.run([sys.executable, __file__, "--worker", *todo], capture_output=True, text=True,
                           timeout=60 + 20 * len(todo))
        out, tail = r.stdout, (r.stderr or "")[-400:]
    except subprocess.TimeoutExpired as e:
        out = (e.stdout or b"").decode() if isinstance(e.stdout, bytes) else (e.stdout or "")
        tail = "TIMEOUT"
    done = []
    for line in out.splitlines():
        if line.startswith("RESULT"):
            d = json.loads(line[7:])
            n = d.pop("name")
            d["ok"] = bool("err" in d and d["err"] == d["err"] and d["err"] <= d["tol"])
            results[n] = d
            done.append(n)
    for line in out.splitlines():
        if line.startswith("b200:"):
            print("   device:", line)
    remaining = [n for n in todo if n not in done]
    if remaining and len(remaining) == len(todo):
        # the first check itself killed the worker before reporting
        results[remaining[0]] = {"ok": False, "error": "worker died: " + tail}
        remaining = remaining[1:]
    todo = remaining
for n, d in results.items():
    print(f"{n:40s} {'OK  ' if d['ok'] else 'FAIL'} {d.get('err', '')} {d.get('error', '')[-300:]}", flush=True)
os.makedirs(os.path.join(ROOT, "out"), exist_ok=True)
json.dump(results, open(os.path.join(ROOT, "out", "kernel_checks.json"), "w"), indent=1)
print("passed", sum(d["ok"] for d in results.values()), "of", len(results))
