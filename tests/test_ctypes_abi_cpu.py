"""The Python side talks to the CUDA library through hand-written ctypes argtypes tables (ops/__init__.py `_Sig`,
parallel/symm.py `_sigs` / `_vmm_sigs`).  A mismatch in COUNT or KIND against the `extern "C"`
declaration does not fail loudly -- arguments are just reinterpreted.  This test parses every `extern "C" int tepd_*(...)`
in ops/csrc/*.cu and compares it parameter by parameter with what the Python modules install.  Static check only: it says
nothing about whether the VALUES passed at the call sites are the right ones."""
import ctypes
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _c_decls():
    decls = {}
    for path in glob.glob(os.path.join(ROOT, "tepdist_b200", "ops", "csrc", "*.cu")):
        src = open(path).read()
        for m in re.finditer(r'extern\s+"C"\s+int\s+(tepd_\w+)\s*\(([^)]*)\)\s*\{', src, re.S):
            name, params = m.group(1), m.group(2)
            kinds = []
            for prm in [p.strip() for p in params.replace("\n", " ").split(",") if p.strip()]:
                stars = prm.count("*")
                base = re.sub(r"\bconst\b|\*", " ", prm)
                base = " ".join(base.split()[:-1])            # drop the parameter name
                if stars >= 2 or re.search(r"\*\s*const\s*\*", prm):
                    kinds.append("pp")
                elif stars == 1:
                    kinds.append("p")
                elif base == "long long":
                    kinds.append("ll")
                elif base == "int":
                    kinds.append("i")
                elif base == "float":
                    kinds.append("f")
                elif base == "unsigned long long":
                    kinds.append("ull")
                else:
                    kinds.append("?" + base)
            assert name not in decls, f"{name} declared twice"
            decls[name] = kinds
    return decls


def _kind(t):
    if t is ctypes.c_void_p:
        return "p"
    if t is ctypes.c_int:
        return "i"
    if t is ctypes.c_longlong:
        return "ll"
    if t is ctypes.c_float:
        return "f"
    if t in (ctypes.c_ulonglong, ctypes.c_ulong) and ctypes.sizeof(t) == 8:
        return "ull"
    if isinstance(t, type) and issubclass(t, ctypes._Pointer):
        # POINTER(c_void_p) = an array of pointers / an out-pointer to a pointer ("pp"); POINTER(<scalar>) = a plain out-parameter
        return "pp" if t._type_ is ctypes.c_void_p else "p"
    return "?" + repr(t)


class _FakeFn:
    def __init__(self):
        self.argtypes, self.restype = None, None


class _FakeLib:
    def __init__(self):
        self.fns = {}

    def __getattr__(self, name):
        if name.startswith("tepd_"):
            return self.fns.setdefault(name, _FakeFn())
        raise AttributeError(name)


def _python_tables():
    from tepdist_b200 import ops
    from tepdist_b200.parallel import symm
    tables = {n: getattr(ops._Sig, n) for n in dir(ops._Sig) if n.startswith("tepd_")}
    lib = _FakeLib()
    symm._sigs(lib)
    symm._vmm_sigs(lib)
    for name, fn in lib.fns.items():
        assert name not in tables, f"{name} has two argtypes tables"
        tables[name] = fn.argtypes
    return tables


def test_every_ctypes_table_matches_its_c_declaration():
    decls, tables = _c_decls(), _python_tables()
    assert len(decls) >= 35, sorted(decls)
    problems = []
    for name, argtypes in sorted(tables.items()):
        if name not in decls:
            problems.append(f"{name}: Python declares argtypes but the library has no such extern \"C\" entry")
            continue
        want, got = decls[name], [_kind(t) for t in argtypes]
        if len(want) != len(got):
            problems.append(f"{name}: C takes {len(want)} parameters, ctypes table has {len(got)}")
            continue
        for k, (w, g) in enumerate(zip(want, got)):
            # a `void* const*` / `T**` parameter must be passed as POINTER(c_void_p); plain pointers as c_void_p
            if w != g:
                problems.append(f"{name}: parameter {k} is '{w}' in C but '{g}' in the ctypes table")
    assert not problems, "\n".join(problems)


def test_every_kernel_entry_point_has_a_ctypes_table():
    """Entry points without an argtypes table would be called with ctypes' default int conversion (truncates 64-bit pointers)."""
    decls, tables = _c_decls(), _python_tables()
    internal = {"tepd_make_tmap_bf16_3d", "tepd_make_tmap_bshd", "tepd_make_tmap_3d"}       # called from C++ only
    missing = sorted(set(decls) - set(tables) - internal)
    assert not missing, missing
