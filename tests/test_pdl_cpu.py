"""CPU: the bookkeeping of the programmatic-dependent-launch suite (tests/test_pdl_gpu.py).

- every C-ABI entry point that launches work has a row in the PDL contract table, so a new entry point without one
  fails here, before any GPU run;
- the test hooks report their argument errors before any device call;
- VILA_B200_NO_PDL: read once per process, '1' as its first character turns PDL off.
"""
import ctypes as C
import os
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent

# entry points that launch nothing: library plumbing and the partition query
NON_LAUNCHING = {"vila_last_error", "vila_abi_version", "vila_set_workspace", "vila_device_info",
                 "vila_gemv_batch_partition"}


def _header_functions():
    text = (ROOT / "include" / "vila_b200.h").read_text()
    return set(re.findall(r"^(?:int|const char\*)\s+(vila_[a-z0-9_]+)\s*\(", text, flags=re.M))


def test_every_launching_entry_point_has_a_pdl_row():
    from tests import test_pdl_gpu as T
    declared = _header_functions()
    assert {"vila_linear", "vila_gemv", "vila_prefix_block_hash", "vila_test_pdl_late"} <= declared
    rows = {entry for entry, _, _ in T.CASES.values()}
    launching = declared - NON_LAUNCHING
    missing = sorted(launching - rows - T.NOT_CONSUMERS)
    assert not missing, f"entry points without a row in tests/test_pdl_gpu.py CASES: {missing}"
    assert not (rows - declared), sorted(rows - declared)
    assert not (T.NOT_CONSUMERS - declared)


def test_every_row_states_a_contract():
    """the kernels that may work before their wait have cases with the static arguments on and off"""
    from tests import test_pdl_gpu as T
    ids = [T._case_id(k) for k in T.CASES]
    assert len(ids) == len(set(ids))
    for stem in ("linear-skinny", "linear-stream-k", "linear-pair", "linear-split-k2", "qkv_rope",
                 "gemv_case-bf16-4608-3584-norm", "gemv_case-fp8", "gemv_case-w4", "gemv_batch_case-fp8",
                 "gemv_batch_case-w4"):
        hits = [i for i in ids if stem in i]
        assert any(i.endswith("False") or "-False-" in i for i in hits), stem
        assert any(i.endswith("True") or "-True-" in i for i in hits), stem
    for regime in ("head", "cluster", "split"):
        assert f"decode_attention-{regime}" in ids


def _lib():
    from vila_b200 import _lib
    return _lib.load()


def test_late_producer_argument_errors_come_first():
    lib = _lib()
    cases = [
        ((None, 0, None, 0, -1), "delay_ns"),
        ((None, 0, None, 0, 2_000_001), "delay_ns"),
        ((None, 65, None, 0, 1000), "n_snap"),
        ((None, 0, None, -1, 1000), "n_late"),
        ((None, 1, None, 0, 1000), "copy list"),
        ((None, 0, None, 2, 1000), "copy list"),
        ((None, 0, 12, 0, 1000), "misaligned"),
    ]
    for args, what in cases:
        rc = lib.vila_test_pdl_late(*args, None)
        msg = lib.vila_last_error().decode()
        assert rc == 1 and what in msg and "CUDA" not in msg, (args, rc, msg)


def test_probe_argument_errors_come_first():
    lib = _lib()
    for flag, seen in ((8, None), (None, 8), (6, 8)):
        rc = lib.vila_test_pdl_probe(flag, seen, None, None)
        msg = lib.vila_last_error().decode()
        assert rc == 1 and "test_pdl_probe" in msg, (flag, seen, rc, msg)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_hooks_need_a_device_after_their_checks():
    lib = _lib()
    assert lib.vila_test_pdl_late(None, 0, None, 0, 1000, None) == 3
    assert b"no CUDA device" in lib.vila_last_error()
    buf = (C.c_int32 * 4)()
    assert lib.vila_test_pdl_probe(C.addressof(buf), C.addressof(buf) + 8, None, None) == 3


def _pdl_in_child(value):
    env = {k: v for k, v in os.environ.items() if k != "VILA_B200_NO_PDL"}
    if value is not None:
        env["VILA_B200_NO_PDL"] = value
    code = ("from vila_b200 import ops; import os; a = ops.pdl_enabled(); "
            "os.environ['VILA_B200_NO_PDL'] = '0' if a is False else '1'; "
            "print(int(a), int(ops.pdl_enabled()))")
    res = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stderr
    first, again = res.stdout.split()
    assert first == again, "VILA_B200_NO_PDL must be read once per process"
    return first == "1"


@pytest.mark.parametrize("value,on", [(None, True), ("1", False), ("0", True), ("", True), ("10", False),
                                      ("yes", True), ("true", True)])
def test_no_pdl_parsing(value, on):
    """PDL is off exactly when VILA_B200_NO_PDL starts with '1'; the value is read once per process"""
    assert _pdl_in_child(value) is on
