"""Runs a script written against the reference's ``uccl`` package on this library: installs the module aliases
(`uccl_b200.compat`) and executes the script as ``__main__``.  A manual tool: run it on
scripts from a checkout of the reference (the test-suite does not run them).

    python tests/run_reference_script.py /path/to/reference/p2p/tests/test_engine_send.py [args...]
"""
import os
import runpy
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import uccl_b200.compat  # noqa: E402

uccl_b200.compat.install()
if os.environ.get("UCCL_B200_ALIAS_TOPLEVEL_UTILS") == "1":
    # p2p/tests/test_util_interval_tree.py imports the sibling file p2p/utils.py as a top-level module
    sys.modules["utils"] = sys.modules["uccl.utils"]
sys.argv = sys.argv[1:]
runpy.run_path(sys.argv[0], run_name="__main__")
