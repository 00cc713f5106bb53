"""The test modules stand on their own: none imports another test module (helpers shared between them live in the
non-test modules beside them)."""
import ast
import glob
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def test_no_test_module_imports_another():
    found = []
    for path in sorted(glob.glob(os.path.join(HERE, "*.py"))):
        with open(path, encoding="utf-8") as f:
            tree = ast.parse(f.read(), path)
        for node in ast.walk(tree):
            if isinstance(node, ast.Import):
                names = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom) and node.level == 0 and node.module:
                names = [node.module]
            else:
                continue
            found += [f"{os.path.basename(path)}:{node.lineno} imports {m}" for m in names
                      if m.split(".")[0].startswith("test_")]
    assert not found, found
