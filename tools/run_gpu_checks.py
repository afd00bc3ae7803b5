#!/usr/bin/env python
"""Run tests/kernel_checks.py checks on the GPU, crash-isolated.

A worker process runs checks one after another and prints one JSON line per check; if a kernel
traps (CUDA context dies) or a check hangs, the parent records it and restarts a worker on the
remaining checks.  Results -> bench_out/kernel_checks.json.
"""
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def worker(names):
    import torch  # noqa
    from tests.kernel_checks import CHECKS

    for n in names:
        print(json.dumps({"start": n}), flush=True)
        t0 = time.time()
        try:
            r = CHECKS[n]()
            torch.cuda.synchronize()
            r["check"] = n
            r["secs"] = round(time.time() - t0, 2)
        except Exception as e:  # noqa
            r = {"check": n, "ok": False, "exception": f"{type(e).__name__}: {e}"[:600]}
            print(json.dumps(r), flush=True)
            if "CUDA" in str(e) or "cuda" in str(e):
                sys.exit(3)  # context is probably dead
            continue
        print(json.dumps(r), flush=True)


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--worker":
        worker(sys.argv[2:])
        return
    from tests.kernel_checks import CHECKS

    names = [a for a in sys.argv[1:] if not a.startswith("-")] or list(CHECKS)
    per_check_timeout = float(os.environ.get("STB_CHECK_TIMEOUT", "150"))
    results = []
    remaining = list(names)
    while remaining:
        proc = subprocess.Popen([sys.executable, __file__, "--worker", *remaining], stdout=subprocess.PIPE,
                                stderr=subprocess.PIPE, text=True, cwd=str(ROOT))
        current = None
        import threading

        err_lines = []
        threading.Thread(target=lambda: err_lines.extend(proc.stderr.readlines()), daemon=True).start()
        deadline = [time.time() + per_check_timeout + 120]

        def watchdog():
            while proc.poll() is None:
                if time.time() > deadline[0]:
                    proc.kill()
                    return
                time.sleep(1)

        threading.Thread(target=watchdog, daemon=True).start()
        for line in proc.stdout:
            line = line.strip()
            if not line.startswith("{"):
                if line:
                    err_lines.append(line + "\n")
                continue
            rec = json.loads(line)
            if "start" in rec:
                current = rec["start"]
                deadline[0] = time.time() + per_check_timeout
                continue
            results.append(rec)
            print(("PASS " if rec.get("ok") else "FAIL ") + json.dumps(rec), flush=True)
            if rec["check"] in remaining:
                remaining.remove(rec["check"])
            current = None
        proc.wait()
        if current is not None and current in remaining:
            rec = {"check": current, "ok": False, "crashed": True, "returncode": proc.returncode,
                   "stderr_tail": "".join(err_lines)[-1500:]}
            results.append(rec)
            print("CRASH " + json.dumps(rec), flush=True)
            remaining.remove(current)
        elif proc.returncode not in (0, 3) and remaining:
            # died before starting anything
            rec = {"check": remaining[0], "ok": False, "crashed": True, "returncode": proc.returncode,
                   "stderr_tail": "".join(err_lines)[-1500:]}
            results.append(rec)
            print("CRASH " + json.dumps(rec), flush=True)
            remaining.pop(0)
    out = ROOT / "bench_out"
    out.mkdir(exist_ok=True)
    (out / "kernel_checks.json").write_text(json.dumps(results, indent=1))
    npass = sum(1 for r in results if r.get("ok"))
    print(f"SUMMARY {npass}/{len(results)} passed; failed: {[r['check'] for r in results if not r.get('ok')]}")


if __name__ == "__main__":
    main()
