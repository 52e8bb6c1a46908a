"""TEST INFRASTRUCTURE: run the emulated tests of tests/test_evaluate_cpu.py (the evaluation records kernel and
Waterworld's heuristic with one norm per env) against AddressSanitizer / UBSan builds of the emulator library, as
tests/emu/sanitize.py does for tests/test_emulated_kernels.py and tests/test_heuristics.py:

    python tests/emu/sanitize_evaluate.py [address|undefined]

Out-of-bounds reads and writes of the records kernel on its carry, record and input buffers, and of the env-norm
policy kernel, show up as sanitizer reports.  Not part of the default test run (an extra build)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

CODE = r'''
import sys
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
from emu import driver
driver._libs[()] = driver.open_lib(%(lib)r)
import pytest
sys.exit(pytest.main([%(testfile)r, "-x", "-q", "-k", "emulated or statistics or c_entry_points", "-p", "no:cacheprovider"]))
'''


def main():
    san = sys.argv[1] if len(sys.argv) > 1 else "address"
    from emu import build_emu
    build_emu.CXXFLAGS += ["-fsanitize=" + san, "-fno-omit-frame-pointer", "-fno-sanitize-recover=all"]
    lib = build_emu.build(["-DMADRL_SANITIZER_%s=1" % san.upper()], force=True)
    env = dict(os.environ)
    rt = {"address": "libasan.so", "undefined": "libubsan.so"}[san]
    for cxx in (os.environ.get("CXX", "g++"), "g++", "/usr/bin/g++"):   # the first compiler that ships the runtime
        path = subprocess.run([cxx, "-print-file-name=" + rt], capture_output=True, text=True).stdout.strip()
        if os.path.isabs(path):
            env["LD_PRELOAD"] = path
            break
    else:
        raise SystemExit("no %s found" % rt)
    env["ASAN_OPTIONS"] = "detect_leaks=0:detect_stack_use_after_return=0:halt_on_error=1"
    code = CODE % dict(tests=os.path.join(ROOT, "tests"), root=ROOT, lib=lib,
                       testfile=os.path.join(ROOT, "tests", "test_evaluate_cpu.py"))
    return subprocess.call([sys.executable, "-c", code], env=env, cwd=ROOT)


if __name__ == "__main__":
    sys.exit(main())
