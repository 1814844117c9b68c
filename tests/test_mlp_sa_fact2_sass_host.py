"""What ptxas makes of mlp_sa_fact2_kernel (no device needed): mlp_tc.cu compiled for sm_90a with the library's own
flags, every instantiation checked for serialised wgmma, spills and the number of warpgroup waits in its SASS.

A wgmma whose accumulator ptxas cannot prove untouched by other code gets its own warpgroup.arrive and a full wait
(warnings C7519 / C7520), and the tensor core then runs one MMA at a time.  The kernel keeps every wgmma width a
compile-time constant so that this does not happen; these tests catch a change that brings it back."""
import os
import re
import shutil
import subprocess

import pytest

from pvn3d_b200 import build

KERNEL = "mlp_sa_fact2_kernel"   # mangled names contain it; mlp_sa_fact2w_kernel does not
CUOBJDUMP = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")

pytestmark = pytest.mark.skipif(not (os.path.exists(build.NVCC) and os.path.exists(CUOBJDUMP)),
                                reason="needs nvcc and cuobjdump")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    out = tmp_path_factory.mktemp("sass")
    cubin = str(out / "mlp_tc.cubin")
    r = subprocess.run([build.NVCC, *build.FLAGS, "-Xptxas", "-v", "-cubin", os.path.join(build.CSRC, "mlp_tc.cu"),
                        "-o", cubin], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([CUOBJDUMP, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    yield r.stderr, sass
    shutil.rmtree(out, ignore_errors=True)


def _ptxas_props(log):
    """mangled kernel name -> (registers, spill store bytes, spill load bytes) from the -Xptxas -v log"""
    props, name = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            props.setdefault(name, [0, 0, 0])[1:] = [int(m.group(1)), int(m.group(2))]
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            props.setdefault(name, [0, 0, 0])[0] = int(m.group(1))
    return {k: tuple(v) for k, v in props.items()}


def _sass_functions(sass):
    """mangled kernel name -> its SASS text"""
    parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
    return dict(zip(parts[1::2], parts[2::2]))


def test_no_serialised_wgmma(compiled):
    log, _ = compiled
    bad = [line for line in log.splitlines() if re.search(r"C75(19|20)", line) and KERNEL in line]
    assert not bad, "\n".join(bad)


def test_no_spills(compiled):
    log, _ = compiled
    props = {k: v for k, v in _ptxas_props(log).items() if KERNEL in k}
    assert len(props) >= 4, log[-2000:]
    for name, (regs, st, ld) in props.items():
        assert st == 0 and ld == 0, f"{name}: {regs} registers, {st} B spill stores, {ld} B spill loads"


def test_warpgroup_waits_per_commit_group(compiled):
    _, sass = compiled
    funcs = {k: v for k, v in _sass_functions(sass).items() if KERNEL in k}
    assert len(funcs) >= 4
    for name, text in funcs.items():
        hgmma = len(re.findall(r"\bHGMMA\.", text))
        depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR", text))
        assert hgmma > 0, name
        assert 2 * depbar < hgmma, f"{name}: {depbar} WARPGROUP.DEPBAR for {hgmma} HGMMA"
