"""Compare the SASS of the kernels two builds share, per kernel.

    python scripts/sass_compare.py OLD.o|OLD.so NEW.o|NEW.so [--filter gemv_ring_kernel]

Runs `cuobjdump -sass` on both files, drops the instruction addresses and the column padding (it follows the length of the
kernel names in the file), and reports for every kernel present in OLD whether NEW holds identical instructions and
encodings.  Exits 1 if any shared kernel differs.  Used to show that a change leaves existing instantiations untouched,
e.g. the 8-row ring GEMV kernels when the 16-row ones were added next to them.
"""
import argparse
import re
import subprocess
import sys


def kernels(path):
    text = subprocess.run(["cuobjdump", "-sass", path], check=True, capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        if cur is not None:
            line = re.sub(r"/\*[0-9a-f]{4}\*/", "", line)          # instruction address
            line = " ".join(line.split())
            if line:
                cur.append(line)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--filter", default="", help="only kernels whose mangled name contains this")
    a = ap.parse_args()
    old, new = kernels(a.old), kernels(a.new)
    bad = 0
    for name in sorted(old):
        if a.filter not in name:
            continue
        status = "missing" if name not in new else "identical" if old[name] == new[name] else "DIFFERENT"
        bad += status != "identical"
        print(f"{status:10s} {len(old[name]):6d} lines  {name}")
    for name in sorted(set(new) - set(old)):
        if a.filter in name:
            print(f"{'new':10s} {len(new[name]):6d} lines  {name}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
