"""The suite's layout: test modules share helpers through tests/_*.py, never through each other.

A bar or helper that lives in one test module and is imported by another changes two modules'
assertions when one is edited; a helper copied into several modules drifts. Both are read from
the source with ast, so nothing under test is imported here."""
import ast
import collections
import os

TESTS = os.path.dirname(os.path.abspath(__file__))


def _modules():
    return sorted(f for f in os.listdir(TESTS) if f.endswith('.py'))


def _tree(name):
    with open(os.path.join(TESTS, name)) as f:
        return ast.parse(f.read(), filename=name)


def _imported(node):
    """Every dotted name an import statement can load: the modules, and module.name for 'from' imports (a name may be
    a submodule).  A relative import is taken relative to tests."""
    if isinstance(node, ast.Import):
        return [a.name for a in node.names]
    if isinstance(node, ast.ImportFrom):
        mod = node.module or ''
        if node.level:
            mod = 'tests' + ('.' + mod if mod else '')
        return [mod] + ['%s.%s' % (mod, a.name) for a in node.names]
    return []


def _strip_docstring(node):
    body = node.body
    if body and isinstance(body[0], ast.Expr) and isinstance(body[0].value, ast.Constant) \
            and isinstance(body[0].value.value, str):
        body = body[1:]
    return body


def _without_docstrings(node):
    """ast.unparse of a top-level def or class with the docstrings of it and its members dropped."""
    node = ast.parse(ast.unparse(node)).body[0]         # a copy
    for n in ast.walk(node):
        if isinstance(n, (ast.FunctionDef, ast.AsyncFunctionDef, ast.ClassDef)):
            n.body = _strip_docstring(n) or [ast.Pass()]
    return ast.unparse(node)


def test_no_test_module_imports_another():
    bad = []
    for name in _modules():
        if not name.startswith('test_'):
            continue
        for node in ast.walk(_tree(name)):            # function bodies included
            if any(m.startswith('tests.test_') for m in _imported(node)):
                bad.append('%s:%d: %s' % (name, node.lineno, ast.unparse(node)))
    assert not bad, 'test modules import other test modules:\n' + '\n'.join(bad)


def test_no_helper_is_defined_twice():
    seen = collections.defaultdict(list)
    for name in _modules():
        for node in _tree(name).body:
            if isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef, ast.ClassDef)):
                seen[(node.name, _without_docstrings(node))].append(name)
    dup = ['%s in %s' % (k[0], ', '.join(v)) for k, v in sorted(seen.items()) if len(v) > 1]
    assert not dup, 'same top-level definition in more than one file under tests/:\n' + '\n'.join(dup)
