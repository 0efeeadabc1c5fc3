"""Device-timed throughput of every bench config in one compact table (no CPU arms):
    python tools/quick_bench.py [label]      (HWYB200_LIB selects an alternative build of the library)"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
label = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("HWYB200_LIB", "default")
out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--no-cpu-baseline", "--steps", "40"]
                     + (["--configs", os.environ["QB_CONFIGS"]] if os.environ.get("QB_CONFIGS") else []),
                     capture_output=True, text=True)
if out.returncode != 0:
    print(label, "FAILED", out.stderr[-600:])
    raise SystemExit(1)
d = json.loads(out.stdout.strip().splitlines()[-1])
print(label, " ".join(f"{c['id']}={c['value']/1e6:.3f}M(e2e {c['e2e']['value']/1e6:.3f}M, kern {c['roofline']['kernel_ms']:.3f}ms)" for c in d["configs"]))
