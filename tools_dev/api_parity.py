"""Name-level parity of the Python API with the reference's pybind layer: every enum (and its values), every module
function, every class and every bound method / property name of the reference's HugeCTR/include/pybind/*.hpp must
exist somewhere in this package.  The names are read from tests/golden/reference_pybind_api.json; `--extract DIR`
regenerates that file from a reference checkout's pybind header directory.  `--json` for machine output.

  python tools_dev/api_parity.py
"""
import glob
import importlib
import inspect
import json
import os
import pkgutil
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "reference_pybind_api.json")
DEAD = {"Holder", "set_callback"}          # a test stub in training_callback.hpp that does not compile against the interface


def extract(txt):
    """names of the pybind layer (the text of all its headers)"""
    enums = {m.group(1): re.findall(r'\.value\("(\w+)"', m.group(2))
             for m in re.finditer(r'enum_<[^>]+>\(\s*\w+\s*,\s*"(\w+)"\)(.*?);', txt, re.S)}
    fns = set(re.findall(r'\bm(?:odule)?\.def\(\s*"(\w+)"', txt)) | set(re.findall(r'\b\w+\.def\(\s*"(Create\w+)"', txt))
    classes = set(re.findall(r'class_<[^;]*?>\s*(?:\w+\s*)?\(\s*\w+\s*,\s*"(\w+)"', txt, re.S)) - DEAD
    members = set(re.findall(r'\.def(?:_readonly|_readwrite|_property_readonly|_static)?\(\s*"([a-zA-Z_0-9]+)"', txt)) - DEAD
    # keyword-argument names of the bound constructors / factory functions (pybind11::arg("...") lists)
    ctor = {}
    for m in re.finditer(r'm\.def\(\s*"(\w+)"(.*?)\);', txt, re.S):
        ctor[m.group(1)] = re.findall(r'pybind11::arg\("(\w+)"\)', m.group(2))
    for m in re.finditer(r'class_<[^;]*?>\s*(?:\w+\s*)?\(\s*\w+\s*,\s*"(\w+)"\)(.*?);\n', txt, re.S):
        a = re.findall(r'pybind11::arg\("(\w+)"\)', m.group(2).split('.def("')[0])
        if a:
            ctor.setdefault(m.group(1), a)
    return {"enums": enums, "functions": sorted(fns), "classes": sorted(classes), "members": sorted(members),
            "ctor_kwargs": ctor}


def ours():
    import hugectr_b200 as h
    have = set(dir(h))
    for m in pkgutil.walk_packages(h.__path__, "hugectr_b200."):
        try:
            mod = importlib.import_module(m.name)
        except Exception:
            continue
        for n in dir(mod):
            have.add(n)
            o = getattr(mod, n)
            if isinstance(o, type):
                have |= set(dir(o))
                try:
                    have |= set(inspect.signature(o.__init__).parameters)
                except (TypeError, ValueError):
                    pass
    return h, have


def main(argv):
    if "--extract" in argv:
        src = argv[argv.index("--extract") + 1]
        txt = "".join(open(f).read() for f in sorted(glob.glob(os.path.join(src, "*.hpp"))))
        with open(GOLDEN, "w") as f:
            json.dump(extract(txt), f, indent=0, sort_keys=True)
        print("wrote", GOLDEN)
        return 0
    with open(GOLDEN) as f:
        ref = json.load(f)
    h, have = ours()
    rep = {"enums": 0, "enum_values": 0, "functions": 0, "classes": 0, "members": 0, "missing": []}
    for name, vals in ref["enums"].items():
        rep["enums"] += 1
        rep["enum_values"] += len(vals)
        cls = getattr(h, name, None)
        if cls is None:
            rep["missing"].append(f"enum {name}")
        else:
            rep["missing"] += [f"{name}.{v}" for v in vals if not hasattr(cls, v)]
    fns = ref["functions"]
    rep["functions"] = len(fns)
    rep["missing"] += [f"function {n}" for n in fns if n not in have]
    classes = ref["classes"]
    rep["classes"] = len(classes)
    rep["missing"] += [f"class {n}" for n in classes if n not in have and not hasattr(h, n)]   # (lazy module attributes)
    members = ref["members"]
    rep["members"] = len(members)
    rep["missing"] += [f"member {n}" for n in members if n not in have]
    rep["kwargs"] = 0
    import hugectr_b200.tools as tools
    for name, a in sorted(ref["ctor_kwargs"].items()):
        o = getattr(h, name, None) or getattr(tools, name, None)
        if o is None:
            continue
        sig = inspect.signature(o.__init__ if isinstance(o, type) else o)
        varkw = any(p_.kind == p_.VAR_KEYWORD for p_ in sig.parameters.values())
        for x in a:
            rep["kwargs"] += 1
            if x not in sig.parameters and not (varkw and x == "lambda"):     # `lambda` is a Python keyword: via **kw
                rep["missing"].append(f"{name}({x}=...)")
    if "--json" in argv:
        print(json.dumps(rep))
    else:
        print(f"{rep['enums']} enums / {rep['enum_values']} values, {rep['functions']} module functions, "
              f"{rep['classes']} classes, {rep['members']} bound members, {rep['kwargs']} constructor keyword names: missing {rep['missing'] or 'none'}")
    return 1 if rep["missing"] else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
