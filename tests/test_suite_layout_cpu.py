"""The shape of the suite: test modules share code only through the helper modules (kernel_harness.py, engine_harness.py,
abi_model.py, util.py), never by importing one another, and every module imports without the library, so that a checkout without a
built libhawq_b200.so still collects and runs its CPU tests."""
import ast
import glob
import os
import subprocess
import sys

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
MODULES = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(TESTS, "*.py"))
                 if os.path.basename(p) not in ("__init__.py", "conftest.py"))


def test_no_test_module_imports_another():
    bad = []
    for name in (m for m in MODULES if m.startswith("test_")):
        for node in ast.walk(ast.parse(open(os.path.join(TESTS, name + ".py")).read())):
            if isinstance(node, ast.Import):
                mods = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom):
                pkg = ("tests." + (node.module or "")).rstrip(".") if node.level else node.module or ""
                mods = [pkg] + [pkg + "." + a.name for a in node.names]
            else:
                continue
            bad += ["%s.py:%d imports %s" % (name, node.lineno, m) for m in mods if m.startswith("tests.test_")]
    assert not bad, bad


def test_every_module_imports_without_the_library(tmp_path):
    code = ("import importlib\nfrom hawq_b200 import _lib\n_lib.LIB_PATH = %r\n"
            "for m in %r:\n    importlib.import_module('tests.' + m)\nassert _lib._lib is None\n") % (str(tmp_path / "missing.so"), MODULES)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
