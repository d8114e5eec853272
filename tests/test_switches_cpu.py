"""The run-time switches are pinned: the SRL_* environment variables the sources read are exactly the rows of DESIGN.md's
"Run-time switches" table.  A new switch has to be documented there; a switch that is no longer read has to leave the table.
Reads the sources; no GPU needed."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C_EXT = ('.cu', '.cuh', '.h')
# reads only: getenv("SRL_X") in C++; os.environ.get / os.getenv / os.environ[...] (not an assignment) in Python
C_READ = re.compile(r'\bgetenv\(\s*"(SRL_\w+)"')
PY_READ = re.compile(r'''\bos\.(?:environ\.get|getenv)\(\s*['"](SRL_\w+)['"]|\bos\.environ\[\s*['"](SRL_\w+)['"]\s*\](?!\s*=[^=])''')


def reads(text, c_source):
    if c_source:
        return set(C_READ.findall(text))
    return {a or b for a, b in PY_READ.findall(text)}


def sources():
    """(path, is C++) of every source the project runs: the package with its CUDA sources, the oracle, the tests, the entry points"""
    here = os.path.abspath(__file__)
    for top in ('scalerl_b200', 'oracle', 'tests', 'include'):
        for d, dirs, files in os.walk(os.path.join(ROOT, top)):
            dirs[:] = [x for x in dirs if x not in ('_ref', 'build', '__pycache__')]
            for f in files:
                p = os.path.join(d, f)
                if f.endswith('.py') and p != here:
                    yield p, False
                elif f.endswith(C_EXT):
                    yield p, True
    for f in ('bench.py', '__graft_entry__.py'):
        yield os.path.join(ROOT, f), False


def documented():
    with open(os.path.join(ROOT, 'DESIGN.md')) as fh:
        text = fh.read()
    assert '\n## Run-time switches\n' in text, 'DESIGN.md has no "Run-time switches" section'
    section = text.split('\n## Run-time switches\n', 1)[1].split('\n## ', 1)[0]
    return set(re.findall(r'^\| `(SRL_\w+)` \|', section, re.M))


def test_switch_table_matches_the_sources():
    found = {}
    for path, c_source in sources():
        with open(path, errors='replace') as fh:
            for name in reads(fh.read(), c_source):
                found.setdefault(name, []).append(os.path.relpath(path, ROOT))
    table = documented()
    undocumented = {k: v for k, v in found.items() if k not in table}
    assert not undocumented, f'switches read but missing from the DESIGN.md table: {undocumented}'
    assert not table - set(found), f'DESIGN.md lists switches no source reads: {sorted(table - set(found))}'
    assert any(c for p, c in sources()) and 'SRL_PDL' in found      # the scan did reach the CUDA sources


def test_the_scan_sees_reads_and_ignores_writes():
    assert reads('static const bool on = [] { const char* e = getenv("SRL_NEW"); return e != nullptr; }();', True) == {'SRL_NEW'}
    assert reads("x = os.environ.get('SRL_A', '1'); y = os.getenv(\"SRL_B\"); z = os.environ['SRL_C']; w = os.environ['SRL_D'] == '1'",
                 False) == {'SRL_A', 'SRL_B', 'SRL_C', 'SRL_D'}
    assert reads("os.environ['SRL_E'] = '1'; os.environ.setdefault('SRL_F', '1'); env['SRL_G'] = '0'", False) == set()
