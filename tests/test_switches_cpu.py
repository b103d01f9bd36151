"""CPU-only: the environment switches.  The table in INTEGRATION.md section 4 lists exactly the RTEN_B200_* variables
the library reads with getenv, and every one of them has a user: the public header documents it, or a test or tool
sets it.  A switch added without a row, a row left behind by a removed switch, and a switch that nothing sets fail
here."""
import pathlib
import re

HERE = pathlib.Path(__file__).resolve()
ROOT = HERE.parent.parent
_READ = re.compile(r'getenv\("(RTEN_B200_[A-Z0-9_]+)"\)')
_ROW = re.compile(r"^\| `(RTEN_B200_[A-Z0-9_]+)` \|", re.M)
_NAME = re.compile(r"RTEN_B200_[A-Z0-9_]+")


def read_by_library():
    """{switch: the source files that read it}"""
    found = {}
    for p in sorted((ROOT / "rten_b200" / "csrc").rglob("*")):
        if p.suffix in (".cu", ".cuh", ".h"):
            for name in _READ.findall(p.read_text()):
                found.setdefault(name, set()).add(p.name)
    return found


def table_rows():
    """the switch of every row of the table in INTEGRATION.md section 4, in order"""
    text = (ROOT / "INTEGRATION.md").read_text()
    assert "\n## 4." in text, "INTEGRATION.md has no section 4"
    return _ROW.findall(text.split("\n## 4.", 1)[1].split("\n## ", 1)[0])


def named_by_users():
    """every RTEN_B200_* name in the public header and in the Python files under tests/ (but this one) and tools/"""
    files = [ROOT / "include" / "rten_b200.h"]
    files += [p for d in ("tests", "tools") for p in sorted((ROOT / d).rglob("*.py")) if p.resolve() != HERE]
    return {name for p in files for name in _NAME.findall(p.read_text())}


def test_table_lists_every_switch_the_library_reads():
    read, rows = read_by_library(), table_rows()
    assert rows, "INTEGRATION.md section 4 has no table of RTEN_B200_* switches"
    assert len(rows) == len(set(rows)), f"rows listed twice: {sorted({r for r in rows if rows.count(r) > 1})}"
    missing = {name: sorted(read[name]) for name in sorted(set(read) - set(rows))}
    stale = sorted(set(rows) - set(read))
    assert not missing, f"switches read by the library with no row in INTEGRATION.md section 4 (name: read in): {missing}"
    assert not stale, f"rows of INTEGRATION.md section 4 for switches the library no longer reads: {stale}"


def test_every_switch_has_a_user():
    switches = set(read_by_library()) | set(table_rows())
    unused = sorted(switches - named_by_users())
    assert not unused, f"switches that include/rten_b200.h does not document and no test or tool sets: {unused}"
