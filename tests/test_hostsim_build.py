"""The cache of the CPU tier's host libraries (tests/hostsim): the shims and the specialised programs of SpecProgram.

A stale library means a CPU test checks old code, so the key must cover every file a library is built from, including every
header it can include: csrc/*.h, csrc/*.cuh and include/rbd_b200.h, whose ABI structs the shims fill in.  CPU only, and nothing
is compiled: g++ and the loader are stubbed out, and edits to a file's bytes are made in the reader, never in the sources."""
import os
import tempfile
import types

import pytest

from tests import hostsim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rigidbodydynamics", "jl_b200", "csrc")
SHIMS = sorted(f[:-4] for f in os.listdir(os.path.join(ROOT, "tests", "hostsim")) if f.endswith(".cpp"))
HEADERS = {os.path.realpath(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))} | {
    os.path.realpath(os.path.join(ROOT, "include", "rbd_b200.h"))}


class Fake:
    """hostsim's compile step with g++ and the loader stubbed out and the temporary directory under ``tmp``."""

    def __init__(self, monkeypatch, tmp):
        monkeypatch.setattr(tempfile, "tempdir", str(tmp))
        self.reads, self.edit, self.text, self.gxx, self.loaded, self._bytes = set(), None, "// program\n", [], [], {}
        monkeypatch.setattr(hostsim, "_read", self._read)
        monkeypatch.setattr(hostsim.subprocess, "check_call", self._gxx)
        monkeypatch.setattr(hostsim, "_load", self._load)
        monkeypatch.setattr(hostsim, "spec_source", lambda *a, **k: (self.text, {}))

    def _load(self, so):
        self.loaded.append(so)
        return types.SimpleNamespace(rbd_spec_cpu=types.SimpleNamespace())

    def _read(self, path):
        path = os.path.realpath(path)
        self.reads.add(path)
        if path not in self._bytes:
            with open(path, "rb") as f:
                self._bytes[path] = f.read()
        return self._bytes[path] + (b"\n// edited\n" if path == self.edit else b"")

    def _gxx(self, argv):
        self.gxx.append(argv)
        open(argv[argv.index("-o") + 1], "wb").close()

    def path(self, target):
        """The library ``target`` (a shim's name, or "SpecProgram") resolves to."""
        if target != "SpecProgram":
            return hostsim.build(target)
        hostsim.SpecProgram(None)
        return self.loaded[-1]


TARGETS = SHIMS + ["SpecProgram"]


@pytest.fixture
def fake(monkeypatch, tmp_path):
    return Fake(monkeypatch, tmp_path)


def test_every_shim_is_a_target():
    assert {"hostsim", "hostsim_adjoint", "hostsim_loops"} <= set(SHIMS)


@pytest.mark.parametrize("target", TARGETS)
def test_key_inputs_cover_every_header(fake, target):
    fake.path(target)
    assert HEADERS <= fake.reads
    if target != "SpecProgram":
        assert os.path.realpath(os.path.join(ROOT, "tests", "hostsim", target + ".cpp")) in fake.reads
        assert os.path.realpath(os.path.join(CSRC, "rbd_model.cpp")) in fake.reads


@pytest.mark.parametrize("target", TARGETS)
def test_every_key_input_changes_the_key(fake, monkeypatch, target):
    p0 = fake.path(target)
    inputs = sorted(fake.reads)
    for f in inputs:
        fake.edit = f
        assert fake.path(target) != p0, f
    fake.edit = None
    assert fake.path(target) == p0
    if target == "SpecProgram":
        fake.text = "// another program\n"
        assert fake.path(target) != p0
        fake.text = "// program\n"
    flags = "SPEC_FLAGS" if target == "SpecProgram" else "SHIM_FLAGS"
    monkeypatch.setattr(hostsim, flags, getattr(hostsim, flags) + ["-g"])
    assert fake.path(target) != p0


@pytest.mark.parametrize("target", ["hostsim", "hostsim_task_vjp", "SpecProgram"])
def test_cache_is_per_user_and_reused(fake, tmp_path, target):
    d = os.path.join(str(tmp_path), f"rbd_hostsim_{os.getuid()}")
    assert hostsim.cache_dir() == d
    p = fake.path(target)
    assert os.path.dirname(p) == d and os.listdir(tmp_path) == [os.path.basename(d)]
    assert len(fake.gxx) == 1 and fake.gxx[0][fake.gxx[0].index("-o") + 1].startswith(os.path.join(d, ""))
    assert fake.path(target) == p and len(fake.gxx) == 1           # same bytes: no second compile
