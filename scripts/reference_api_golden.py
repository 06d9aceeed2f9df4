#!/usr/bin/env python
"""Extract the public Python surface of a BaguaSys/bagua checkout into ``tests/golden/reference_api.json``.

For every module of the reference's ``bagua`` package: its public top-level functions and classes, and the parameter names
(in order) of every public function and public method / ``__init__`` of its public classes.  ``tests/test_api_surface.py``
checks the ``bagua`` alias package of this project against this file, so the tests need no copy of the reference.

    python scripts/reference_api_golden.py /path/to/bagua-checkout > tests/golden/reference_api.json
"""
import ast
import json
import os
import sys


def extract(root: str) -> dict:
    modules = {}
    pkg = os.path.join(root, "bagua")
    for d, _, files in sorted(os.walk(pkg)):
        for f in sorted(files):
            if not f.endswith(".py"):
                continue
            path = os.path.join(d, f)
            mod = os.path.relpath(path, root)[:-3].replace(os.sep, ".")
            mod = mod[: -len(".__init__")] if mod.endswith(".__init__") else mod
            try:
                tree = ast.parse(open(path).read())
            except SyntaxError:
                continue
            names = [n.name for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and not n.name.startswith("_")]
            sigs = {}
            for n in tree.body:
                if isinstance(n, ast.FunctionDef) and not n.name.startswith("_"):
                    items = [(n.name, n)]
                elif isinstance(n, ast.ClassDef) and not n.name.startswith("_"):
                    items = [(f"{n.name}.{k.name}", k) for k in n.body if isinstance(k, ast.FunctionDef) and (k.name == "__init__" or not k.name.startswith("_"))]
                else:
                    continue
                for name, node in items:
                    sigs[name] = [a.arg for a in node.args.posonlyargs + node.args.args if a.arg not in ("self", "cls")]
            modules[mod] = {"names": names, "signatures": sigs}
    return {"source": "BaguaSys/bagua python package (bagua/**/*.py), extracted by scripts/reference_api_golden.py", "modules": modules}


if __name__ == "__main__":
    json.dump(extract(sys.argv[1]), sys.stdout, indent=1, sort_keys=True)
    sys.stdout.write("\n")
