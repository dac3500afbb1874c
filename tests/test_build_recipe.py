"""The one build recipe behind the default library, the one-stage-ring stress library and the experiment variants
(gaustudio_b200/build.py::_build), checked without nvcc or a GPU: build.py is pointed at an empty copy of the source
tree and at a stub nvcc that records each command line and creates the file named by -o.

- every source is compiled with exactly [NVCC, *FLAGS, "-c", src, "-o", obj], the stress and variant builds adding only
  their -D flags;
- every output is rebuilt when include/gsr.h or a csrc/ header is newer than it, and only then;
- no object file outlives the build."""
import importlib.util
import os

import pytest

from gaustudio_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRESS_DEFINES = ["-DGSR_NSTAGE=1", "-DGSR_RB=32"]
VARIANT = "cluster_scan"
STUB = """#!/bin/sh
for a in "$@"; do printf '%s\\n' "$a"; done > "$(mktemp "{calls}/XXXXXX")"
prev=
for a in "$@"; do
  if [ "$prev" = "-o" ]; then : > "$a"; fi
  prev=$a
done
echo "ptxas info    : stub"
"""


@pytest.fixture
def tree(tmp_path, monkeypatch):
    """<tmp>/gaustudio_b200/csrc with empty files of the real names, <tmp>/include/gsr.h, and the stub nvcc; all sources
    dated well in the past so that a freshly linked output is newer than each."""
    csrc = tmp_path / "gaustudio_b200" / "csrc"
    csrc.mkdir(parents=True)
    (tmp_path / "include").mkdir()
    deps = [tmp_path / "include" / "gsr.h"] + [csrc / f for f in os.listdir(build.CSRC)
                                                 if f.endswith((".cu", ".cuh", ".h"))]
    for d in deps:
        d.write_text("")
        os.utime(d, (1e9, 1e9))
    calls = tmp_path / "calls"
    calls.mkdir()
    nvcc = tmp_path / "nvcc"
    nvcc.write_text(STUB.format(calls=calls))
    nvcc.chmod(0o755)
    here = str(tmp_path / "gaustudio_b200")
    monkeypatch.setattr(build, "NVCC", str(nvcc))
    monkeypatch.setattr(build, "HERE", here)
    monkeypatch.setattr(build, "CSRC", str(csrc))
    monkeypatch.setattr(build, "LIB", os.path.join(here, "libgsr_b200.so"))
    monkeypatch.setattr(build, "STRESS_LIB", os.path.join(here, "libgsr_b200_stress.so"))
    return tmp_path


def _calls(tree):
    """The command lines the stub recorded since the last call, compiles first in SOURCES order, then the link."""
    out = []
    for f in (tree / "calls").iterdir():
        out.append([build.NVCC] + f.read_text().splitlines())
        f.unlink()
    compiles = [c for c in out if "-c" in c]
    compiles.sort(key=lambda c: build.SOURCES.index(os.path.basename(c[c.index("-c") + 1])))
    return compiles + [c for c in out if "-c" not in c]


def _variants():
    spec = importlib.util.spec_from_file_location("build_variants", os.path.join(ROOT, "tools", "build_variants.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _run(kind):
    """Build one output through its public entry point -> (output path, the -D flags it adds)."""
    if kind == "default":
        return build.build_library(), []
    if kind == "stress":
        return build.build_stress_variant(), STRESS_DEFINES
    bv = _variants()
    bv.build([VARIANT])
    return os.path.join(build.HERE, "variants", f"libgsr_{VARIANT}.so"), bv.VARIANTS[VARIANT]


@pytest.mark.parametrize("kind", ["default", "stress", "variant"])
def test_each_source_is_compiled_with_the_library_flags_plus_only_the_defines(tree, kind):
    out, defines = _run(kind)
    calls = _calls(tree)
    assert len(calls) == len(build.SOURCES) + 1
    objs = []
    for s, cmd in zip(build.SOURCES, calls):
        objs.append(cmd[-1])
        assert cmd == [build.NVCC, *build.FLAGS, *defines, "-c", os.path.join(build.CSRC, s), "-o", objs[-1]]
    assert calls[-1] == [build.NVCC, "-shared", "-Xlinker", f"-soname={os.path.basename(out)}", "-o", out, *objs,
                         "-lcudart", "-ldl"]
    assert os.path.exists(out)
    log = os.path.join(build.CSRC, "ptxas.log") if kind == "default" else os.path.splitext(out)[0] + ".ptxas.log"
    assert open(log).read().count("ptxas info    : stub") == len(build.SOURCES)


@pytest.mark.parametrize("touched", ["include/gsr.h", "gaustudio_b200/csrc/gsr_internal.cuh"])
@pytest.mark.parametrize("kind", ["default", "stress", "variant"])
def test_an_output_older_than_a_header_is_rebuilt(tree, kind, touched):
    out, _ = _run(kind)
    _calls(tree)
    assert _run(kind)[0] == out and _calls(tree) == [], "an up-to-date output was rebuilt"
    t = os.path.getmtime(out) + 10
    os.utime(tree / touched, (t, t))
    _run(kind)
    assert len(_calls(tree)) == len(build.SOURCES) + 1, f"{kind} build not redone after {touched} changed"


def test_no_object_file_outlives_the_build(tree):
    for kind in ("default", "stress", "variant"):
        _run(kind)
        objs = [c[-1] for c in _calls(tree) if "-c" in c]
        assert objs and not any(os.path.exists(o) for o in objs)
        assert not any(os.path.exists(os.path.dirname(o)) for o in objs)
    assert not list(tree.rglob("*.o"))
