"""CPU tests (no GPU): SCS_B200_G_REUSE, the switch that makes every scs_solve re-solve g (DESIGN.md section 3.2,
"Reusing g"), as each library flavour reads it. The environment is read at every call, so one process can run both
arms of an A/B comparison."""
import pytest

from scs_b200 import capi

FLAVOURS = [dict(), dict(spectral=True), dict(long=True), dict(spectral=True, long=True)]


@pytest.mark.parametrize("flavour", FLAVOURS, ids=lambda f: "-".join(f) or "default")
def test_switch(flavour, monkeypatch):
    lib = capi.load(**flavour)
    monkeypatch.delenv("SCS_B200_G_REUSE", raising=False)
    assert lib.scs_b200_g_reuse() == 1
    for value, reuse in (("0", 0), ("1", 1), ("", 1)):
        monkeypatch.setenv("SCS_B200_G_REUSE", value)
        assert lib.scs_b200_g_reuse() == reuse, value
