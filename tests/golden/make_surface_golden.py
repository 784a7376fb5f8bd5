"""Build tests/golden/api_surface.json: the public Python surface of the reference that the host layer must keep.

Needs a checkout of theislab/dca:  python tests/golden/make_surface_golden.py /path/to/dca-checkout

Read with `ast` (TensorFlow / scanpy are not importable here, and nothing of the reference is executed):
  dca/api.py:19-45       dca(...)           parameter names, order and default values
  dca/train.py:35-39     train(...)         parameter names, order and default values
  dca/network.py:44-59   Autoencoder.__init__
  dca/network.py:763-768 AE_types keys
  dca/__main__.py:21-136 CLI flags with their defaults (literal defaults only)
"""
import ast
import json
import os

import sys

REF = os.path.join(sys.argv[1] if len(sys.argv) > 1 else ".", "dca")
HERE = os.path.dirname(os.path.abspath(__file__))


def _lit(node):
    try:
        return ast.literal_eval(node)
    except Exception:
        return "<expr:%s>" % ast.unparse(node)


def _params(fn):
    a = fn.args
    names = [x.arg for x in a.args]
    defaults = [None] * (len(names) - len(a.defaults)) + [_lit(d) for d in a.defaults]
    has_default = [False] * (len(names) - len(a.defaults)) + [True] * len(a.defaults)
    return [{"name": n, "has_default": h, "default": d} for n, h, d in zip(names, has_default, defaults)] + \
           ([{"name": "**" + a.kwarg.arg, "has_default": False, "default": None}] if a.kwarg else [])


def _function(path, name, cls=None):
    tree = ast.parse(open(path).read())
    for node in ast.walk(tree):
        if cls and isinstance(node, ast.ClassDef) and node.name == cls:
            for sub in node.body:
                if isinstance(sub, ast.FunctionDef) and sub.name == name:
                    return _params(sub)
        if not cls and isinstance(node, ast.FunctionDef) and node.name == name:
            return _params(node)
    raise KeyError(name)


def _ae_types(path):
    tree = ast.parse(open(path).read())
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "AE_types" for t in node.targets):
            return [ast.literal_eval(k) for k in node.value.keys]
    raise KeyError("AE_types")


def _cli_flags(path):
    flags = []
    for node in ast.walk(ast.parse(open(path).read())):
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "add_argument":
            names = [ast.literal_eval(x) for x in node.args if isinstance(x, ast.Constant)]
            kw = {k.arg: _lit(k.value) for k in node.keywords if k.arg in ("default", "dest", "action", "type")}
            flags.append({"names": names, **{k: (v if not callable(v) else str(v)) for k, v in kw.items()}})
    return flags


def main():
    out = {"source": "theislab/dca @ 6abd124 (read with ast, not executed)",
           "api.dca": _function(os.path.join(REF, "api.py"), "dca"),
           "train.train": _function(os.path.join(REF, "train.py"), "train"),
           "network.Autoencoder.__init__": _function(os.path.join(REF, "network.py"), "__init__", cls="Autoencoder"),
           "network.AE_types": _ae_types(os.path.join(REF, "network.py")),
           "cli": _cli_flags(os.path.join(REF, "__main__.py"))}
    with open(os.path.join(HERE, "api_surface.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True, default=str)
    print("wrote api_surface.json:", {k: (len(v) if isinstance(v, list) else v) for k, v in out.items()})


if __name__ == "__main__":
    main()
