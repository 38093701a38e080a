import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: the library is built for sm_90a)")
    config.addinivalue_line("markers", "ref: needs oracle/_ref/libstrelka_ref.so (the reference compiled by oracle/build_ref.sh)")


def pytest_collection_modifyitems(config, items):
    from reflib import have_ref

    if have_ref():
        return
    skip = pytest.mark.skip(reason="oracle/_ref/libstrelka_ref.so not built (reference tree absent)")
    for it in items:
        if "ref" in it.keywords:
            it.add_marker(skip)
