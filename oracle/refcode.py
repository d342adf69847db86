"""The one way into a checkout of the reference (locuslab/icnn) -- TEST INFRASTRUCTURE ONLY.

The golden generators run the reference's own code: modules that import under numpy / scipy are imported unchanged
(``load``); functions, classes, methods and statement ranges of files that import TensorFlow at module level are cut
out with ``ast`` and exec'd unmodified in a namespace the caller fills (``extract``, ``run_statements``).  The
checkout is found through $ICNN_REFERENCE_DIR; ``available()`` says whether every file the generators read is there.
"""
import ast
import contextlib
import importlib.util
import io
import os

import numpy as np

DIR = os.environ.get("ICNN_REFERENCE_DIR", "")
FILES = ("lib/bundle_entropy.py", "lib/bundle_entropy_dual.py", "RL/src/bundle_entropy.py", "RL/src/icnn.py",
         "multi-label-cls/icnn_ebundle.py", "multi-label-cls/icnn-back.py", "multi-label-cls/ebundle-vs-gd.py",
         "completion/icnn_ebundle.py", "completion/icnn.back.py")


def path(rel):
    return os.path.join(DIR, rel)


def available():
    return bool(DIR) and all(os.path.isfile(path(f)) for f in FILES)


def load(name, rel):
    """Import the reference file ``rel`` unchanged as a module called ``name``."""
    spec = importlib.util.spec_from_file_location(name, path(rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _parse(rel):
    with open(path(rel)) as fh:
        src = fh.read()
    return ast.parse(src), src.splitlines()


def _find(body, kind, name):
    node = [n for n in body if isinstance(n, kind) and n.name == name]
    assert len(node) == 1, name
    return node[0]


def _exec(rel, body, namespace):
    exec(compile(ast.Module(body=body, type_ignores=[]), path(rel), "exec"), namespace)
    return namespace


def extract(rel, names, namespace):
    """exec the definitions ``names`` of the reference file ``rel``, verbatim, in ``namespace`` and return it.  A name
    is a top-level function or class, or 'Class.method': that method alone, bound under its own name."""
    tree, _ = _parse(rel)
    body = []
    for name in names:
        if "." in name:
            cls, meth = name.split(".")
            body.append(_find(_find(tree.body, ast.ClassDef, cls).body, ast.FunctionDef, meth))
        else:
            body.append(_find(tree.body, (ast.ClassDef, ast.FunctionDef), name))
    return _exec(rel, body, namespace)


def run_statements(rel, method, first, last, namespace):
    """exec the statements of ``method`` ('Class.method') of the reference file ``rel``, from the one whose first line
    reads ``first`` through the one whose first line reads ``last`` (both stripped), in ``namespace``."""
    tree, lines = _parse(rel)
    cls, meth = method.split(".")
    stmts = _find(_find(tree.body, ast.ClassDef, cls).body, ast.FunctionDef, meth).body
    text = [lines[s.lineno - 1].strip() for s in stmts]
    assert text.count(first) == 1 and text.count(last) == 1, (method, first, last)
    return _exec(rel, stmts[text.index(first):text.index(last) + 1], namespace)


@contextlib.contextmanager
def quiet():
    """Reference code prints progress and trips numpy's floating-point warnings: silence both, return its stdout."""
    with contextlib.redirect_stdout(io.StringIO()) as out, np.errstate(all="ignore"):
        yield out
