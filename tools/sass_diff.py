"""Compare the SASS of the engine library built from two source trees, function by function.

    python tools/sass_diff.py OLD_ROOT NEW_ROOT [extra nvcc flags, e.g. -DLLQ16_BLOCK=128 or -DLLQ16_TIMING]

Builds lifelike_agility_and_play_b200/csrc/llq_cuda.cu of each tree with __graft_entry__.NVCC_FLAGS + -Xptxas -v (+ the extra
flags) in a temporary directory, splits `cuobjdump -sass` by function and prints the functions whose instructions differ or that
exist in one build only, with both builds' registers and spill bytes.  Exit status 1 when any function differs.  A tree of an
earlier commit: `git worktree add /tmp/parent HEAD~1`.  Needs nvcc and cuobjdump, no GPU."""
import os
import re
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from __graft_entry__ import NVCC_FLAGS  # noqa: E402

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def build(root, extra, out):
    """{function: SASS text}, {function: (registers, spill stores, spill loads)} of root's engine library"""
    lib = os.path.join(out, "lib.so")
    log = subprocess.run([os.path.join(CUDA, "bin", "nvcc")] + NVCC_FLAGS + ["-Xptxas", "-v"] + extra +
                         ["-o", lib, os.path.join(root, "lifelike_agility_and_play_b200", "csrc", "llq_cuda.cu")],
                         check=True, capture_output=True, text=True).stderr
    res = {}
    for name, body in re.findall(r"Compiling entry function '(\w+)'(.*?)(?=Compiling entry function|\Z)", log, re.S):
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", body)
        res[name] = (int(re.search(r"Used (\d+) registers", body).group(1)),) + tuple(int(x) for x in spill.groups())
    sass = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", lib], check=True, capture_output=True, text=True).stdout
    # (cuobjdump pads its columns to the widest line of the whole file: compare the tokens, not the padding)
    return {f: " ".join(body.split()) for f, body in re.findall(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\n\s*\.{10}|\Z)", sass, re.S)}, res


def main():
    old_root, new_root, extra = sys.argv[1], sys.argv[2], sys.argv[3:]
    with tempfile.TemporaryDirectory() as tmp:
        (a, ra), (b, rb) = [build(root, extra, tempfile.mkdtemp(dir=tmp)) for root in (old_root, new_root)]
    differ = sorted(f for f in set(a) | set(b) if a.get(f) != b.get(f))
    for f in sorted(set(a) | set(b)):
        print("%-9s %s  regs/spill stores/loads %s -> %s" % ("DIFFERS" if f in differ else "same", f, ra.get(f), rb.get(f)))
    print("%d of %d functions differ" % (len(differ), len(set(a) | set(b))))
    return 1 if differ else 0


if __name__ == "__main__":
    sys.exit(main())
