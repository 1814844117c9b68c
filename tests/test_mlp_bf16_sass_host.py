"""What ptxas makes of the bf16 forms in mlp_tc.cu (no device needed): the dense layer kernel, FP1's bf16 row store and
the bf16 gather, compiled for sm_90a with the library's own flags.

Every instantiation must have 0 spill bytes and no serialised wgmma (C7519 / C7520), and the dense kernel's MMAs must
be bf16 HGMMA: a change that quietly falls back to tf32 MMAs, or that makes a wgmma width a run-time choice again, fails
here."""
import re

# the compile fixture, its helpers and its skip condition (needs nvcc and cuobjdump)
from test_mlp_sa_fact2_sass_host import _ptxas_props, _sass_functions, compiled, pytestmark  # noqa: F401

DENSE = "mlp_dense_bf16_kernel"
BF16_KERNELS = (DENSE, "mlp_fp_fact2_kernelILi2E", "gather_pixel_rows_bf16_kernel")


def _bf16_names(names):
    return [k for k in names if any(s in k for s in BF16_KERNELS)]


def test_every_bf16_instantiation_is_compiled(compiled):  # noqa: F811
    log, _ = compiled
    names = _bf16_names(_ptxas_props(log))
    # dense: {store bf16, store f32, sum-pool} x wgmma N {16, 32, 64, 128}; FP1 rows; gather from f32 and from bf16
    assert len([k for k in names if DENSE in k]) == 12, names
    assert len(names) == 15, names


def test_no_spills(compiled):  # noqa: F811
    log, _ = compiled
    props = {k: v for k, v in _ptxas_props(log).items() if k in _bf16_names([k])}
    assert props
    for name, (regs, st, ld) in props.items():
        assert st == 0 and ld == 0, f"{name}: {regs} registers, {st} B spill stores, {ld} B spill loads"


def test_no_serialised_wgmma(compiled):  # noqa: F811
    log, _ = compiled
    bad = [line for line in log.splitlines() if re.search(r"C75(19|20)", line) and _bf16_names([line])]
    assert not bad, "\n".join(bad)


def test_dense_kernel_runs_bf16_hgmma(compiled):  # noqa: F811
    _, sass = compiled
    funcs = {k: v for k, v in _sass_functions(sass).items() if DENSE in k}
    assert len(funcs) == 12
    for name, text in funcs.items():
        hgmma = re.findall(r"\bHGMMA\.\S+", text)
        assert hgmma, name
        assert all(".BF16" in h for h in hgmma), f"{name}: {sorted(set(hgmma))}"
        # one width per instantiation: four MMAs per K chunk, one commit group each
        depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR", text))
        assert 2 * depbar < len(hgmma), f"{name}: {depbar} WARPGROUP.DEPBAR for {len(hgmma)} HGMMA"
