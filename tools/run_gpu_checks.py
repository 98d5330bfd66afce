"""Run every kernel check in its own process (a trapped kernel kills only its own CUDA context).
Writes gpurun_out/kernel_checks.json.  Usage: python tools/run_gpu_checks.py [name-substring ...]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--one":
        import kernel_checks as kc
        import model_checks as mc

        fn = getattr(kc, sys.argv[2], None) or getattr(mc, sys.argv[2])
        t0 = time.time()
        res = fn()
        import torch

        torch.cuda.synchronize()
        print("RESULT " + json.dumps({"ok": True, "res": res, "sec": round(time.time() - t0, 2)}))
        return
    import kernel_checks as kc
    import model_checks as mc

    names = [c.__name__ for c in kc.ALL_CHECKS + mc.ALL_CHECKS]
    filt = sys.argv[1:]
    if filt:
        names = [n for n in names if any(f in n for f in filt)]
    out_dir = os.path.join(ROOT, "gpurun_out")
    os.makedirs(out_dir, exist_ok=True)
    results = {}
    env = dict(os.environ, DK_DUMP_DIR=os.path.join(out_dir, "dumps"))
    for n in names:
        try:
            p = subprocess.run([sys.executable, __file__, "--one", n], capture_output=True, text=True, timeout=400,
                               env=env)
            line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            if line:
                results[n] = json.loads(line[-1][7:])
            else:
                tail = (p.stdout + "\n" + p.stderr).strip().splitlines()[-12:]
                results[n] = {"ok": False, "rc": p.returncode, "tail": tail}
        except subprocess.TimeoutExpired:
            results[n] = {"ok": False, "timeout": True}
        print(n, json.dumps(results[n])[:600], flush=True)
    with open(os.path.join(out_dir, "kernel_checks.json"), "w") as f:
        json.dump(results, f, indent=1)
    bad = [n for n, r in results.items() if not r.get("ok")]
    print(f"{len(results) - len(bad)}/{len(results)} checks passed; failed: {bad}")


if __name__ == "__main__":
    main()
