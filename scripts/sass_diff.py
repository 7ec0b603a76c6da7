#!/usr/bin/env python
r"""Compare the SASS of the kernels in spades_b200/csrc/build/count.o (or another object: --obj covfilter) with a build of another
commit (default: the last commit whose kernels ran on the GPU). Used when refactoring without GPU access: identical SASS of the default kernels == nothing to re-verify.
    python scripts/sass_diff.py [--obj NAME] <commit> ['regex=>replacement' ...]   (renames applied to the old mangled names, e.g. new template arguments)
    python scripts/sass_diff.py 8f22764 'local_sort3_kILi([12])EEE=>local_sort3_kILi\1ELi11ELi2048EEE' 'local_sort3_kILi([34])EEE=>local_sort3_kILi\1ELi11ELi1024EEE' \
        'levelA_scatter_roll_kILi(\d)ELb(\d)EEE(.*)PKtjjj=>levelA_scatter_roll_kILi\1ELb\2ELb0EEE\3PKtjjjj' 'refine_kILi(\d)ELb(\d)EEE=>refine_kILi\1ELb\2ELb0EEE'
"""
import re
import subprocess
import sys
import tempfile


def sass(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    # an anonymous namespace is mangled with hashes of the source's path: the same kernel built in another directory
    out = re.sub(r"_GLOBAL__N__[0-9a-f]{8}_(\d+_\w+?)_[0-9a-f]{8}", r"_GLOBAL__N__\1", out)
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1); funcs[cur] = []; continue
        if cur and "/*" in line:
            t = re.sub(r"/\*[0-9a-fx]+\*/", "", line).strip()
            if t and not t.startswith("/*"):
                funcs[cur].append(re.sub(r"0x[0-9a-f]+", "X", t))
    return funcs


def main():
    args = sys.argv[1:]
    obj = "count"
    if args[0] == "--obj":
        obj, args = args[1], args[2:]
    commit = args[0]
    renames = [a.split("=>") for a in args[1:]]
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call("git archive %s spades_b200/csrc include | tar -x -C %s" % (commit, d), shell=True)
        subprocess.check_call(["nvcc", "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC", "-c", obj + ".cu",
                               "-o", d + "/old.o"], cwd=d + "/spades_b200/csrc", stderr=subprocess.DEVNULL)
        old = sass(d + "/old.o")
    new = sass("spades_b200/csrc/build/%s.o" % obj)
    bad = 0
    for name, body in sorted(old.items()):
        want = name
        for a, b in renames:
            want = re.sub(a, b, want)
        if want not in new:
            print("gone     ", name); continue
        same = body == new[want]
        bad += not same
        print("%-9s %s" % ("identical" if same else "DIFFERENT", name))
    print("kernels in the old build: %d, in the new build: %d" % (len(old), len(new)))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
