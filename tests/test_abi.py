"""CPU: the C-ABI library builds for sm_90a, loads, and exports exactly the symbols include/esb200.h declares
(no compute calls without a GPU); the product path fails loudly without the library."""
import ctypes
import os

import pytest

from abi_util import header_signatures


def test_library_builds_and_exports_every_declared_symbol():
    from embodiedscan_b200 import _ffi
    from embodiedscan_b200.build import build_library
    path = build_library()
    assert os.path.exists(path)
    handle = ctypes.CDLL(path)
    sigs = header_signatures()
    assert len(sigs) >= 30
    for name in sigs:
        assert hasattr(handle, name), f'{name} declared in include/esb200.h but not exported'
    assert sigs == _ffi.SIGNATURES, 'ctypes binding out of sync with include/esb200.h'


def test_host_only_queries():
    from embodiedscan_b200 import _ffi
    assert _ffi.query('esb_hash_capacity', 1000) == 2048
    assert _ffi.query('esb_hash_capacity', 1) == 1024
    assert _ffi.query('esb_paint_meta_bytes') == 7 * 4 + 8 * 4 + 8 * 9 * 4
    assert _ffi.query('esb_kmap_pairs_workspace_bytes', 27, 1000) > 2 * 27000 * 4


def test_no_cpu_fallback(monkeypatch):
    from embodiedscan_b200 import _ffi
    monkeypatch.setattr(_ffi, '_lib', None)
    monkeypatch.setattr(_ffi, 'LIB_PATH', '/nonexistent/libesb200.so')
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        _ffi.lib()


def test_product_never_imports_oracle():
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'embodiedscan_b200')
    for fn in os.listdir(root):
        if fn.endswith('.py'):
            src = open(os.path.join(root, fn)).read()
            assert 'import oracle' not in src and 'from oracle' not in src, fn
