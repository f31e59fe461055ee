"""CPU: no module under tests/, oracle/ or scripts/ imports a test module (tests/test_*.py).  Shared inputs and helpers
live in the support modules (tests/kernels.py, signals.py, parity.py, golden_cases.py, ...), so that editing one test
cannot change what another test, or a golden generator, computes."""
import ast
import glob
import os

from tests.host_exe import ROOT


def imported_modules(node):
    """Dotted names of the modules an import statement loads: ``tests.x`` for ``from tests import x``, and ``.x`` for a
    relative import."""
    if isinstance(node, ast.Import):
        return [a.name for a in node.names]
    dots = "." * node.level
    if node.module is None or node.module == "tests" and not node.level:
        base = dots or "tests."
        return [base + a.name for a in node.names]
    return [dots + node.module]


def is_test_module(name):
    if name.startswith("."):
        return name.lstrip(".").startswith("test_")
    return name.startswith("tests.test_")


def test_no_module_imports_a_test_module():
    files = [p for d in ("tests", "oracle", "scripts") for p in glob.glob(os.path.join(ROOT, d, "**", "*.py"), recursive=True)]
    assert len(files) > 50, len(files)
    bad = []
    for path in files:
        for node in ast.walk(ast.parse(open(path).read(), path)):
            if isinstance(node, (ast.Import, ast.ImportFrom)):
                bad += ["%s:%d imports %s" % (os.path.relpath(path, ROOT), node.lineno, m)
                        for m in imported_modules(node) if is_test_module(m)]
    assert not bad, "\n".join(bad)
