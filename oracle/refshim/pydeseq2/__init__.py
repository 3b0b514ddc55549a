"""Import shim (TEST INFRASTRUCTURE, golden-data generation only).

Makes a PyDESeq2 source checkout, named by the environment variable PYDESEQ2_SRC,
importable without installing it: the real ``pydeseq2/__init__.py`` calls
``importlib.metadata.version("pydeseq2")`` which fails for an un-installed tree.
Only used by ``oracle/make_golden.py``; nothing on the product path or in the test
suite imports it.
"""
import os

_SRC = os.environ.get("PYDESEQ2_SRC")
if not _SRC:
    raise ImportError("set PYDESEQ2_SRC to a PyDESeq2 0.5.3 source checkout (the directory that holds pydeseq2/)")
__path__ = [os.path.join(_SRC, "pydeseq2")]
__file__ = os.path.join(_SRC, "pydeseq2", "__init__.py")
__version__ = "0.5.3"
