import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "ref: needs oracle/_ref (the compiled unmodified reference)")


def pytest_sessionstart(session):
    """The tests need the in-tree builds (libw2b.so, the CLI, liboracle.so); build them when a fresh
    checkout has none.  (The product itself never builds or falls back at import time.)"""
    need = [os.path.join(ROOT, "word2bits_b200", "libw2b.so"), os.path.join(ROOT, "word2bits_b200", "word2bits"),
            os.path.join(ROOT, "oracle", "liboracle.so")]
    if not all(os.path.exists(p) for p in need):
        import __graft_entry__
        __graft_entry__.build()
