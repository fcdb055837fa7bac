#!/usr/bin/env python
"""Per-function SASS of two builds of the sm_90a kernel library (no GPU needed): which functions of the first are identical
in the second, identical apart from constant-bank parameter offsets, different, or missing.

    python bench/sass_compare.py OLD.so NEW.so

A function is matched by its mangled name without the translation unit's anonymous-namespace hash.  The attention kernels
gained a DROP template parameter and an AttnDropParams kernel parameter, so an old `attn_{fwd,bwd}_kernel<HD, DOC>` is
compared with the new `attn_{fwd,bwd}_kernel<HD, DOC, false>`.
"""
import re
import subprocess
import sys


def functions(path: str) -> dict:
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_(\w+?)_cu_[0-9a-f]{8}", r"\1", m.group(1))
            res[cur] = []
        elif cur and re.search(r"/\*[0-9a-f]{4}\*/", line):
            res[cur].append(re.sub(r"/\*[0-9a-f]{4}\*/", "", line).split(";")[0].strip())
    return res


def main() -> None:
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    params = lambda body: [re.sub(r"c\[0x0\]\[0x[0-9a-f]+\]", "c[0x0][P]", i) for i in body]   # noqa: E731
    counts = {"identical": 0, "parameter offsets only": 0, "different": 0, "missing": 0}
    for name, body in sorted(old.items()):
        cand = re.sub(r"(attn_(?:fwd|bwd)_kernelILi\d+ELb[01])E(.*Params)E$", r"\1ELb0E\2ENS_14AttnDropParamsE", name)
        other = new.get(name, new.get(cand))
        kind = ("missing" if other is None else "identical" if other == body else
                "parameter offsets only" if params(other) == params(body) else "different")
        counts[kind] += 1
        if kind in ("different", "missing"):
            print(f"{kind}: {name}")
    print(f"{len(old)} functions in {sys.argv[1]}: " + ", ".join(f"{v} {k}" for k, v in counts.items()))
    sys.exit(1 if counts["different"] or counts["missing"] else 0)


if __name__ == "__main__":
    main()
