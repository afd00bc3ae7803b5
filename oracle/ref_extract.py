"""Execute selected functions / methods of the reference *verbatim* — TEST INFRASTRUCTURE ONLY.

The reference package cannot be imported in this container (diffusers / accelerate / peft are not
installed, SURVEY.md §8c) but its pure-torch helpers can be lifted out of the source files with
`ast` and exec'ed with only torch/math/random in scope.  Nothing is copied into this repository:
the source text is read at run time from a SimpleTuner checkout named by the SIMPLETUNER_SRC environment
variable (the directory holding the `simpletuner` package), so this module only works where that checkout
exists, and is used by the oracle/make_golden*.py scripts to produce the committed fixtures under tests/golden/.
"""
from __future__ import annotations

import ast
import logging
import math
import os
import random
import types
from pathlib import Path
from typing import Dict, Iterable

import torch
import torch.nn.functional as F

REF_ROOT = Path(os.environ.get("SIMPLETUNER_SRC", "")) / "simpletuner"


def available() -> bool:
    try:
        return bool(os.environ.get("SIMPLETUNER_SRC")) and REF_ROOT.is_dir()
    except OSError:
        return False


def _namespace() -> Dict[str, object]:
    import numbers
    import typing

    ns: Dict[str, object] = {
        "torch": torch, "math": math, "random": random, "F": F,
        "logger": logging.getLogger("ref_extract"), "numbers": numbers,
    }
    ns.update({k: getattr(typing, k) for k in ("Optional", "Any", "Dict", "List", "Tuple", "Union")})
    return ns


def functions(rel_path: str, names: Iterable[str], extra_ns=None) -> Dict[str, object]:
    """Top-level FunctionDefs `names` of reference file `rel_path`, exec'ed as-is."""
    src = (REF_ROOT / rel_path).read_text()
    tree = ast.parse(src)
    want = set(names)
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in want]
    missing = want - {n.name for n in body}
    if missing:
        raise KeyError(f"{rel_path}: functions not found: {sorted(missing)}")
    ns = _namespace()
    if extra_ns:
        ns.update(extra_ns)
    exec(compile(ast.Module(body=body, type_ignores=[]), str(REF_ROOT / rel_path), "exec"), ns)
    return {n: ns[n] for n in want}


def methods(rel_path: str, class_name: str, names: Iterable[str], extra_ns=None) -> type:
    """A dummy class carrying the reference's own method bodies `names` of `class_name`."""
    src = (REF_ROOT / rel_path).read_text()
    tree = ast.parse(src)
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == class_name)
    want = set(names)
    body = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in want]
    missing = want - {n.name for n in body}
    if missing:
        raise KeyError(f"{rel_path}:{class_name}: methods not found: {sorted(missing)}")
    new_cls = ast.ClassDef(name="Lifted" + class_name, bases=[], keywords=[], body=body, decorator_list=[])
    if hasattr(new_cls, "type_params"):
        new_cls.type_params = []
    mod = ast.Module(body=[new_cls], type_ignores=[])
    ast.fix_missing_locations(mod)
    ns = _namespace()
    if extra_ns:
        ns.update(extra_ns)
    exec(compile(mod, str(REF_ROOT / rel_path), "exec"), ns)
    return ns["Lifted" + class_name]
