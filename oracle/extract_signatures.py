#!/usr/bin/env python
"""Writes tests/golden/reference_signatures.json: the public call signatures of the original uccl project that the
API audits in tests/ compare this library against (parameter names only, parsed from its sources).

    python oracle/extract_signatures.py /path/to/uccl [--out tests/golden/reference_signatures.json]
"""
import argparse
import ast
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EP_BUFFERS = ["ep/bench/buffer.py", "thirdparty/DeepEP/deep_ep/buffer.py", "ep/deep_ep_wrapper/deep_ep/buffer.py"]
EP_UTILS = ["ep/bench/utils.py", "thirdparty/DeepEP/deep_ep/utils.py", "thirdparty/DeepEP/tests/utils.py",
            "ep/deep_ep_wrapper/deep_ep/utils.py"]
DEEP_EP_INIT = "ep/deep_ep_wrapper/deep_ep/__init__.py"
P2P_BINDING = "p2p/engine_api.cc"
COLLECTIVE = "p2p/collective.py"


def params(f, drop_self=True):
    a = f.args
    return [x.arg for x in a.posonlyargs + a.args + a.kwonlyargs if not (drop_self and x.arg == "self")]


def buffer_methods(src):
    cls = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.ClassDef) and n.name == "Buffer")
    return {f.name: params(f) for f in cls.body
            if isinstance(f, ast.FunctionDef) and (not f.name.startswith("_") or f.name == "__init__")}


def module_functions(src, drop_self=False):
    return {f.name: params(f, drop_self) for f in ast.parse(src).body
            if isinstance(f, ast.FunctionDef) and not f.name.startswith("_")}


def endpoint_binding(src):
    src = src[src.index("nb::class_<Endpoint>"):] if "nb::class_<Endpoint>" in src else src
    out = {}
    for d in re.split(r'\.def\(\s*"', src)[1:]:
        name = d.split('"', 1)[0]
        if not name.startswith("__"):
            out[name] = re.findall(r'nb::arg\("([a-zA-Z_0-9]+)"\)', d.split(".def(", 1)[0])
    return out


def collective(src):
    tree = ast.parse(src)
    ctx = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "CollectiveContext")
    return {"functions": module_functions(src, drop_self=True),
            "CollectiveContext": {f.name: params(f) for f in ctx.body if isinstance(f, ast.FunctionDef)
                                  and (not f.name.startswith("_") or f.name == "__init__")}}


def deep_ep_all(src):
    for n in ast.walk(ast.parse(src)):
        if isinstance(n, ast.Assign) and any(getattr(t, "id", "") == "__all__" for t in n.targets):
            return ast.literal_eval(n.value)
    raise SystemExit("no __all__ in " + DEEP_EP_INIT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("reference", help="checkout of the original uccl project")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "reference_signatures.json"))
    a = ap.parse_args()

    def read(rel):
        with open(os.path.join(a.reference, rel)) as f:
            return f.read()

    d = {
        "ep_buffer": {p: buffer_methods(read(p)) for p in EP_BUFFERS},
        "ep_utils": {p: module_functions(read(p)) for p in EP_UTILS},
        "deep_ep_all": deep_ep_all(read(DEEP_EP_INIT)),
        "p2p_endpoint": endpoint_binding(read(P2P_BINDING)),
        "collective": collective(read(COLLECTIVE)),
    }
    with open(a.out, "w") as f:
        json.dump(d, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
