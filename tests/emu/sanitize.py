"""TEST INFRASTRUCTURE: run tests/test_emulated_kernels.py and the emulated tests of tests/test_heuristics.py (the
in-kernel policies, the generators) against AddressSanitizer / UBSan builds of the emulator library (kernel source +
host launch code compiled by g++):

    python tests/emu/sanitize.py [address|undefined] [default|experiments]

Out-of-bounds reads and writes of the kernels on the state blob, action and output buffers, shifts
and overflows show up as sanitizer reports.  Not part of the default test run (two extra builds)."""
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
import test_emulated_kernels as T
driver._libs[tuple(sorted(T.VARIANTS[%(variant)r]))] = driver.open_lib(%(lib)r)
import pytest
sys.exit(pytest.main([%(testfile)r, %(heurfile)r, "-x", "-q", "-k", %(variant)r + " or policy or generator or closed_loop",
                      "-p", "no:cacheprovider"]))
'''


def main():
    san = sys.argv[1] if len(sys.argv) > 1 else "address"
    variant = sys.argv[2] if len(sys.argv) > 2 else "default"
    from emu import build_emu
    import test_emulated_kernels as T
    build_emu.CXXFLAGS += ["-fsanitize=" + san, "-fno-omit-frame-pointer", "-fno-sanitize-recover=all"]
    lib = build_emu.build(list(T.VARIANTS[variant]) + ["-DMADRL_SANITIZER_%s=1" % san.upper()], force=True)
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
    code = CODE % dict(tests=os.path.join(ROOT, "tests"), root=ROOT, lib=lib, variant=variant,
                       testfile=os.path.join(ROOT, "tests", "test_emulated_kernels.py"),
                       heurfile=os.path.join(ROOT, "tests", "test_heuristics.py"))
    return subprocess.call([sys.executable, "-c", code], env=env, cwd=ROOT)


if __name__ == "__main__":
    sys.exit(main())
