"""CPU: the written claims that are cheap to verify mechanically — symbol counts quoted in the docs, and that every
`profiles/rNN/...` artefact the docs cite is committed."""
import re
from pathlib import Path

from simpletuner_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent


def test_symbol_counts_in_docs_match_the_abi():
    n = len(_lib.SYMBOLS)
    design = (ROOT / "DESIGN.md").read_text()
    readme = (ROOT / "README.md").read_text()
    assert f"{n} symbols" in design, f"DESIGN.md should quote {n} C-ABI symbols"
    assert f"C ABI ({n} entry points" in readme, f"README.md should quote {n} entry points"


def test_cited_profile_files_exist():
    missing = []
    for doc in ("DESIGN.md", "README.md", "INTEGRATION.md"):
        text = (ROOT / doc).read_text()
        for m in re.finditer(r"profiles/(r0[12])/([A-Za-z0-9_.\-]+\.(?:jsonl|json|csv|log|txt))", text):
            if not (ROOT / "profiles" / m.group(1) / m.group(2)).exists():
                missing.append((doc, m.group(1), m.group(2)))
        if doc.startswith("profiles/"):      # a round's own README may cite its artefacts by bare file name
            rnd = doc.split("/")[1]
            for m in re.finditer(r"`([A-Za-z0-9_.\-]+\.(?:jsonl|json|csv|log|txt))`", text):
                if not (ROOT / "profiles" / rnd / m.group(1)).exists():
                    missing.append((doc, rnd, m.group(1)))
    assert not missing, missing


def test_reference_citations_have_file_and_line():
    """Every C-ABI declaration block cites a reference file:line (include/stb200.h is the boundary document)."""
    header = (ROOT / "include" / "stb200.h").read_text()
    assert len(re.findall(r"[a-z_/]+\.py:\d+", header)) >= 20


def test_cited_repo_files_exist():
    """Every `tests/...py`, `tools/...`, `oracle/...py` and `simpletuner_b200/...` path quoted in the docs is a real file."""
    missing = []
    for doc in ("DESIGN.md", "README.md", "INTEGRATION.md"):
        text = (ROOT / doc).read_text()
        for m in re.finditer(r"`((?:tests|tools|oracle|simpletuner_b200)/[A-Za-z0-9_./\-]+\.(?:py|cu|cuh|sh|pt))(?:::[A-Za-z0-9_\[\]\-., =]+)?`", text):
            if not (ROOT / m.group(1)).exists():
                missing.append((doc, m.group(1)))
    assert not missing, missing
