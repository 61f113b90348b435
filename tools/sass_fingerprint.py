#!/usr/bin/env python
"""Per-kernel fingerprint of the DEVICE code of the product library: md5 of each kernel's SASS instruction stream with addresses,
encodings and the path-dependent anonymous-namespace hash stripped.  Compared with the fingerprints of a build that passed
`pytest -m gpu`, host-only edits, comment edits and explicit re-statements of what the compiler already
generated must leave a kernel's line unchanged (tools/sass_diff.py shows what changed inside a kernel).
usage: sass_fingerprint.py [build-dir]   (default kintinuous_b200/csrc/build)"""
import glob, hashlib, os, re, subprocess, sys

root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
build = sys.argv[1] if len(sys.argv) > 1 else os.path.join(root, "kintinuous_b200", "csrc", "build")
for obj in sorted(glob.glob(os.path.join(build, "*.o"))):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    cur, acc = None, {}
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_", "", m.group(1))
            cur = re.sub(r"_cu_[0-9a-f]{8}", "", cur)
            try:
                cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip() or cur
                cur = re.sub(r"\(anonymous namespace\)::", "", cur).split("(")[0]
            except Exception:
                pass
            acc[cur] = hashlib.md5()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(.*?);", line)
        if m and cur:
            acc[cur].update(m.group(1).strip().encode())
    for k in sorted(acc):
        print(f"{os.path.basename(obj)} {acc[k].hexdigest()[:16]} {k}")
