"""Compare the SASS of two builds function by function: which kernels are identical, which differ, which are new.

Build both trees (``python -m medpy_b200.build``), then

    python tools/compare_sass.py OLD/medpy_b200/lib/obj NEW/medpy_b200/lib/obj

The hashes nvcc puts into anonymous-namespace names depend on the source path; they are normalised, so two checkouts in
different directories compare.  Exits 1 when a kernel present in both builds differs.
"""
import os
import re
import subprocess
import sys

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def functions(obj):
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", m.group(1))
            funcs[cur] = []
        elif cur and re.search(r"/\*[0-9a-f]{4}\*/", line):
            funcs[cur].append(re.sub(r"\s+", " ", line.split(";")[0]).strip())
    return funcs


def main(old_dir, new_dir):
    bad = False
    for name in sorted(os.listdir(new_dir)):
        if not name.endswith(".o"):
            continue
        new = functions(os.path.join(new_dir, name))
        old_path = os.path.join(old_dir, name)
        old = functions(old_path) if os.path.exists(old_path) else {}
        differ = sorted(k for k in old if k in new and old[k] != new[k])
        added = sorted(k for k in new if k not in old)
        gone = sorted(k for k in old if k not in new)
        print("{}: {} identical, {} differ, {} added, {} removed".format(
            name, sum(1 for k in old if old[k] == new.get(k)), len(differ), len(added), len(gone)))
        for k in differ:
            print("  differs:", k)
        bad |= bool(differ)
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) != 3:
        raise SystemExit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))
