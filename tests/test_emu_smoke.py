"""__graft_entry__.smoke() (the one-call end-to-end check on an H100) executed on the CPU emulator: the same function, the same
oracle comparison, the emulated library in place of the CUDA one."""
from tests.cuemu import harness


def test_smoke_entry_point_under_the_emulator(monkeypatch, capsys):
    harness.set_order("fwd")
    harness.emulated_device(monkeypatch)
    import __graft_entry__ as entry
    entry.smoke()
    assert "smoke ok" in capsys.readouterr().out
