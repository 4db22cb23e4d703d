"""CPU: the token of the CG loop's fused K3 + K4 kernel is one per process. It lives in libscs_b200_token.so, which
every library flavour links by soname (scs_b200/csrc/Makefile): no flavour defines it itself, so a process that loads
several flavours, each with RTLD_LOCAL, still has one token."""
import ctypes as C
import os
import subprocess

import pytest

from scs_b200 import capi

HERE = os.path.dirname(capi.LIB_PATH)
TOKEN = os.path.join(HERE, "libscs_b200_token.so")
FLAVOURS = [capi.LIB_PATH, capi.SPECTRAL_LIB_PATH, capi.LONG_LIB_PATH, capi.SPECTRAL_LONG_LIB_PATH,
            capi.LINSYS_LONG_LIB_PATH]
SYMBOLS = {"b200_k34_token_take", "b200_k34_token_give_back"}


def dynsyms(path, *flags):
    out = subprocess.run(["nm", "-D", *flags, path], capture_output=True, text=True, check=True).stdout
    return {line.split()[-1] for line in out.splitlines() if line.strip()}


@pytest.mark.parametrize("path", FLAVOURS, ids=os.path.basename)
def test_every_flavour_takes_the_token_from_the_shared_object(path):
    dyn = subprocess.run(["readelf", "-d", path], capture_output=True, text=True, check=True).stdout
    assert "[libscs_b200_token.so]" in dyn
    assert "$ORIGIN" in dyn
    assert not SYMBOLS & dynsyms(path, "--defined-only")
    assert SYMBOLS <= dynsyms(path, "--undefined-only")


def test_token_is_a_try_lock():
    assert SYMBOLS <= dynsyms(TOKEN, "--defined-only")
    token = C.CDLL(TOKEN)
    assert token.b200_k34_token_take() == 1
    try:
        assert token.b200_k34_token_take() == 0
    finally:
        token.b200_k34_token_give_back()
    assert token.b200_k34_token_take() == 1
    token.b200_k34_token_give_back()
