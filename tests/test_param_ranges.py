"""Seed lengths and scores the Greedy kernels cannot represent are refused before any device work, and kaiju-b200 reads -l, -s, -m and -e
as the reference does (std::stoi into an int, kaiju.cpp:110-166).  CPU only: kj_check_params_c and the CLI's option parsing, which ends
before a context is created."""
import ctypes as C
import os
import subprocess
import pytest
from conftest import ROOT
from helpers import REF_DIR, have_ref

INT32_MAX = 2 ** 31 - 1


@pytest.fixture(scope="module")
def lib(built):
    import kaiju_b200 as kb
    L = kb.lib()
    L.kj_check_params_c.restype = C.c_int; L.kj_check_params_c.argtypes = [C.POINTER(kb.KjParams)]
    return kb, L


@pytest.mark.parametrize("field", ["seed_length", "min_score"])
@pytest.mark.parametrize("mode", ["greedy", "mem"])
def test_check_params_refuses_values_above_int32(lib, field, mode):
    """The kernels compare the seed length and the minimum score as int (kj_core_greedy.h); the reference cannot produce larger values."""
    kb, L = lib
    for v, rc in ((INT32_MAX, 0), (2 ** 31, -1), (2 ** 31 + 1, -1), (2 ** 32 - 1, -1)):
        P = kb.make_params(mode); setattr(P, field, v)
        assert L.kj_check_params_c(C.byref(P)) == rc, (field, mode, v)
        if rc:
            assert b"2^31 - 1" in L.kj_last_error()
    P = kb.make_params("greedy", seed=1, s=1)
    assert L.kj_check_params_c(C.byref(P)) == 0
    P = kb.make_params("greedy"); setattr(P, field, 0)
    assert L.kj_check_params_c(C.byref(P)) == -1


# (option, argument) -> the first line the reference writes to stderr; None: the value is taken (no message)
ARGS = [("-l", "6", "Error: Seed length must be >= 7."), ("-l", "6x", "Error: Seed length must be >= 7."), ("-l", "-3", "Error: Seed length must be >= 7."),
        ("-l", "abc", "Invalid argument in -l abc"), ("-l", "99999999999", "Invalid argument in -l 99999999999"), ("-l", "2147483648", "Invalid argument in -l 2147483648"),
        ("-l", "12x", None), ("-l", " 40", None), ("-l", "2147483647", None),
        ("-s", "0", "Error: Min Score (-s) must be greater than 0."), ("-s", "x1", "Invalid argument in -s x1"), ("-s", "4294967296", "Invalid argument in -s 4294967296"),
        ("-s", "2147483647", None),
        ("-m", "0", "Error: Min fragment length (-m) must be greater than 0."), ("-m", "", "Invalid argument in -m "), ("-m", "3000000000", "Invalid argument in -m 3000000000"),
        ("-m", "9.5", None),
        ("-e", "-1", "Error: Number of mismatches must be >= 0."), ("-e", "x", "Invalid numerical argument in -e x"), ("-e", "1e99999", None)]


def _first_line_and_status(prog, opt, arg):
    # no -t/-f/-i: after the options both programs stop with a usage error, before any file or device is opened
    r = subprocess.run([prog, "-a", "greedy", opt, arg], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)
    return r.stderr.split("\n")[0], r.returncode


@pytest.mark.parametrize("opt,arg,msg", ARGS)
def test_cli_reads_numeric_options_like_the_reference(built, opt, arg, msg):
    cli = os.path.join(ROOT, "kaiju_b200", "kaiju-b200")
    line, rc = _first_line_and_status(cli, opt, arg)
    assert rc == 1
    if msg is None:
        assert line.startswith("Error: Please specify the location of the FMI file"), line      # the option was accepted
    else:
        assert line == msg
    if have_ref():
        rline, rrc = _first_line_and_status(os.path.join(REF_DIR, "kaiju"), opt, arg)
        assert rrc == rc
        assert rline == msg if msg is not None else rline.startswith("Error: Please specify the location of the nodes.dmp file"), rline
