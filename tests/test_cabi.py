"""The C-ABI library loads and exports every entry point include/qrec.h declares.  CPU only:
nothing here launches a kernel."""
import ctypes
import os
import re

from conftest import ROOT


def _declared():
    src = open(os.path.join(ROOT, 'include', 'qrec.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(qrec_[a-z0-9_]+)\s*\(', src)))


def test_every_declared_symbol_is_exported_and_bound():
    from qrec_b200 import _lib
    names = _declared()
    assert len(names) >= 25
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), 'libqrec.so does not export %s' % n
        assert n in _lib.SIGNATURES, 'python binding missing for %s' % n
    assert set(_lib.SIGNATURES) == set(names)


def test_version_and_error_channel():
    from qrec_b200 import engine as E
    from qrec_b200._lib import lib
    assert 'sm_90a' in E.version()
    rc = lib.qrec_mt_seed(None, 0)
    assert rc == -1 and b'null' in lib.qrec_last_error()


def test_product_does_not_touch_oracle():
    """The shipped package must never import oracle/ (parity claims depend on it)."""
    pkg = os.path.join(ROOT, 'qrec_b200')
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cpp', '.h')):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', txt, flags=re.M), f
                assert 'liboracle' not in txt, f


def test_sm90a_only_and_hopper_sass():
    """The cubin inside libqrec.so targets sm_90a and uses the 128-bit vector reduction."""
    import shutil
    import subprocess
    from qrec_b200 import _lib
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip('cuobjdump not available')
    out = subprocess.run([cuobjdump, '-lelf', _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert 'sm_90a' in out and 'sm_100' not in out and 'sm_80' not in out
    sass = subprocess.run([cuobjdump, '-sass', _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert 'REDG.E.ADD.F32x4' in sass          # red.global.add.v4.f32 scatter-add
    assert 'LDG.E.128' in sass                 # 128-bit row gathers


def test_integration_doc_snippets_are_valid_python_and_name_real_symbols():
    """The binding a maintainer would copy from INTEGRATION.md must at least parse, and every C entry
    point it calls must exist in the header."""
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, 'INTEGRATION.md')).read()
    blocks = re.findall(r'```python\n(.*?)```', text, re.S)
    assert blocks
    header = open(os.path.join(root, 'include', 'qrec.h')).read()
    for code in blocks:
        compile(code, 'INTEGRATION.md', 'exec')
        for name in re.findall(r'lib\.(qrec_[a-z0-9_]+)', code):
            assert re.search(r'\b%s\s*\(' % name, header), name
