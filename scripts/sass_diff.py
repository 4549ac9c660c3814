"""Per-kernel SASS comparison between a git revision and the working tree (GPU-less check that a refactor did
not touch the instruction stream of kernels that were already validated on hardware).

    python scripts/sass_diff.py <git-rev>          # e.g. the last commit validated on the GPU

Compiles every csrc/*.cu of <git-rev> into a temp dir, hashes the instruction text of every kernel (addresses and
encodings stripped) and compares with baton_b200/csrc/build/*.o.  Kernels are matched by demangled name, with
template arguments appended at their default value normalised away: trailing `, 0` / `, false` arguments (e.g. the
CONV mode, the SGD and AFFINE epilogue flags) on both sides, and `<true>` on a kernel that was not a template before
(a new `false` instantiation beside it).  New kernels are listed separately."""
import hashlib
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--use_fast_math"]


def kernel_hashes(obj):
    txt = subprocess.run(["cuobjdump", "-sass", obj], stdout=subprocess.PIPE, text=True).stdout
    out = {}
    for fn in re.split(r"\n\s*Function : ", txt)[1:]:
        name = fn.split("\n", 1)[0].strip()
        ins = re.findall(r"/\*[0-9a-f]{4,6}\*/\s+(.*?);", fn)
        out[name] = (hashlib.md5("\n".join(ins).encode()).hexdigest(), len(ins))
    return out


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), stdout=subprocess.PIPE, text=True).stdout.splitlines()
    return dict(zip(names, out))


def canonical(hashes, old_plain=()):
    """demangled name -> hash, appended default-valued template arguments stripped (see the module docstring)"""
    dm = demangle(list(hashes))
    out = {}
    for k, v in hashes.items():
        name = dm[k]
        if name.startswith("void "):
            name = name[5:]
        prev = None
        while prev != name:
            prev = name
            name = re.sub(r", (?:0|false)>\(", ">(", name)
        plain = name.replace("<true>(", "(", 1)
        if plain != name and plain in old_plain:
            name = plain
        assert name not in out, "two kernels normalise to " + name
        out[name] = v
    return out


def main():
    rev = sys.argv[1]
    tmp = tempfile.mkdtemp(prefix="sass_diff_")
    subprocess.run("git archive {} baton_b200/csrc | tar -x -C {}".format(rev, tmp), shell=True, check=True, cwd=ROOT)
    old_dir = os.path.join(tmp, "baton_b200", "csrc")
    procs = []
    for f in sorted(os.listdir(old_dir)):
        if f.endswith(".cu"):
            procs.append(subprocess.Popen(["nvcc"] + FLAGS + ["-c", f, "-o", f[:-3] + ".o"], cwd=old_dir,
                                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL))
    for p in procs:
        p.wait()
    total = same = 0
    for f in sorted(os.listdir(old_dir)):
        if not f.endswith(".o"):
            continue
        new_obj = os.path.join(ROOT, "baton_b200", "csrc", "build", f)
        if not os.path.exists(new_obj):
            print("MISSING OBJECT", f)
            continue
        old = canonical(kernel_hashes(os.path.join(old_dir, f)))
        new = norm = canonical(kernel_hashes(new_obj), old_plain=set(old))
        for k, v in old.items():
            total += 1
            if norm.get(k) == v:
                same += 1
            else:
                print("DIFF  {:14s} {:5d} -> {:5d}  {}".format(f, v[1], norm.get(k, (0, 0))[1], k[:90]))
        fresh = [k for k in new if k not in old]
        if fresh:
            print("NEW   {:14s} {}".format(f, len(fresh)))
    print("kernels in {}: {}   byte-identical instruction stream now: {}".format(rev[:10], total, same))


if __name__ == "__main__":
    main()
