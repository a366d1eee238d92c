"""Launch count of every kernel entry point of libmnn_b200.so over the GPU test suite (needs an H100).

Runs `pytest -m gpu` over tests/: tests/test_gpu_dispatch.py first, in a child process, since it profiles each of its cases
itself and keeps the launches it saw in test_gpu_dispatch.LAUNCHED; then every other module in this process under one
torch.profiler (CUDA activity).  (Short profiling windows opened in a process after one long session lose kernel records, so
the two do not share a process.)  Prints each entry point (tests/test_gpu_dispatch.py's key) with its launch count and the
test KERNEL_TESTS names for it, then the entry points never launched.  Kernels launched by a subprocess of a test (the plugin
tests run the reference executor in one) are not seen.  Exit status 1 if an entry point was never launched or a test failed.

    python tools/kernel_coverage.py [extra pytest arguments]
"""
import json
import os
import subprocess
import sys
import tempfile
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PYTEST_ARGS = ["-m", "gpu", "-q", "-p", "no:cacheprovider"]


def dispatch_module(extra, out_json):
    """child process: the dispatch module alone; its LAUNCHED counter to out_json"""
    import pytest
    rc = pytest.main(PYTEST_ARGS + extra + ["tests/test_gpu_dispatch.py"])
    launched = sys.modules["tests.test_gpu_dispatch"].LAUNCHED
    with open(out_json, "w") as f:
        json.dump([[k[0], list(k[1]), n] for k, n in launched.items()], f)
    return int(rc)


def main(extra):
    from mnn_b200 import build as B
    from tests import test_gpu_dispatch as D

    os.chdir(ROOT)
    entries = D.library_kernels(B.build())
    counts = Counter()
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "launched.json")
        rc_dispatch = subprocess.call([sys.executable, os.path.abspath(__file__), "--dispatch-module", out] + extra)
        if os.path.exists(out):
            with open(out) as f:
                counts.update({(name, tuple(args)): n for name, args, n in json.load(f)})

    import pytest
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rc_rest = pytest.main(PYTEST_ARGS + extra + ["tests", "--ignore=tests/test_gpu_dispatch.py"])
        torch.cuda.synchronize()
    counts.update(D.kernel_key(e.name) for e in prof.events()
                  if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")))

    print(f"\n{'launches':>9}  kernel entry point  [test named in KERNEL_TESTS]")
    for key in sorted(entries, key=lambda k: (k[0], str(k[1]))):
        print(f"{counts[key]:>9}  {key[0]}<{', '.join(str(a) for a in key[1])}>  [{D.KERNEL_TESTS.get(key, '-')}]")
    never = sorted(k for k in entries if not counts[k])
    print(f"\n{len(entries)} entry points, {len(entries) - len(never)} launched, never launched: {never or 'none'}")
    others = sorted(k for k in counts if k not in entries)
    if others:
        print(f"kernels launched that are not entry points of the library (torch's own): {len(others)}")
    print(f"pytest exit codes: test_gpu_dispatch.py {int(rc_dispatch)}, other modules {int(rc_rest)}")
    return 1 if never or rc_rest or rc_dispatch else 0


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--dispatch-module":
        sys.exit(dispatch_module(sys.argv[3:], sys.argv[2]))
    sys.exit(main(sys.argv[1:]))
