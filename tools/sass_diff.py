#!/usr/bin/env python
"""Per-kernel comparison of the SASS of two builds of the same object (addresses, encodings and the path-dependent anonymous-namespace
hash stripped).  Host-only edits, comment edits and explicit re-statements of what the compiler already generated must leave every
kernel identical.   usage: sass_diff.py [--multiset] before.o after.o
--multiset compares each kernel's instructions as a multiset with registers, predicates, branch targets and local-memory offsets
abstracted: a re-statement that only changes register allocation or scheduling passes it, a changed operation or operand does not."""
import collections, re, subprocess, sys


def kernels(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_", "_ANON_", m.group(1))
            cur = re.sub(r"_cu_[0-9a-f]{8}", "_cu_X", cur)
            res[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(.*?);", line)
        if m and cur:
            res[cur].append(m.group(1).strip())
    return res


def abstract(ins):
    ins = re.sub(r"^@!?U?P(\d+|T) ", "@P ", ins.replace(".reuse", ""))
    ins = re.sub(r"\bU?R(\d+|Z)\b", "R", ins)
    ins = re.sub(r"\bU?P(\d+|T)\b", "P", ins)
    ins = re.sub(r"^((@P )?(BRA|BSSY|CALL\.REL(\.NOINC)?|BREAK|BSYNC))\b.*", r"\1", ins)
    ins = re.sub(r"^((@P )?)IMAD\.IADD R, R, 0x1, R$", r"\1IADD3 R, R, R, R", ins)
    return re.sub(r"\[R\+0x[0-9a-f]+\]", "[R+off]", ins)


args = [x for x in sys.argv[1:] if x != "--multiset"]
multiset = len(args) < len(sys.argv) - 1
a, b = kernels(args[0]), kernels(args[1])
if multiset:
    a = {k: sorted(x for x in map(abstract, v) if x != "NOP") for k, v in a.items()}
    b = {k: sorted(x for x in map(abstract, v) if x != "NOP") for k, v in b.items()}
diff = only = 0
for k in sorted(set(a) | set(b)):
    if k not in a or k not in b:
        print("ONLY IN", "before" if k in a else "after", k); only += 1
    elif a[k] != b[k]:
        if multiset:
            ca, cb = collections.Counter(a[k]), collections.Counter(b[k])
            print(f"DIFF  {k}: {len(a[k])} -> {len(b[k])} instructions, {sum((ca - cb).values())} removed, {sum((cb - ca).values())} added")
        else:
            n = sum(1 for x, y in zip(a[k], b[k]) if x != y) + abs(len(a[k]) - len(b[k]))
            print(f"DIFF  {k}: {len(a[k])} -> {len(b[k])} instructions, {n} positions differ")
        diff += 1
common = len(set(a) & set(b))
print(f"{common - diff} of {common} common kernels identical, {only} present in one build only")
sys.exit(1 if diff else 0)
