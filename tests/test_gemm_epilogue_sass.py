"""The GEMM's epilogue variants, read from the built library's SASS (no GPU needed).

The generic epilogue selects a 32-column slot's 16 accumulators at run time (registers cannot be indexed), 16 FSEL per
slot past the first: its FSEL count grows by 16 per 32 columns of tile width. The specialised variants work on
accumulators 0..15 at compile-time indices and move the array down by one slot per iteration, so they add FSELs that do
not depend on the width: ~145, nearly all of them erff's coefficient selects (9 per value) in the GELU-erf variant,
whose slot body evaluates erff for its 16 values. A variant that selected its accumulators at run time, or one unrolled
over the tile, would make the count grow faster (unrolled over the tile the variants made ~20 k-instruction kernels with
1329 FSEL at 256 columns)."""
import re

from test_gemm_sass import library, sass_functions  # noqa: F401  (fixture: both storage-type builds)


def _width(name):
    m = re.search(r"gemm_bf16_wgmma_kernelILi(\d+)ELb([01])E", name)
    return int(m.group(1)), m.group(2) == "1"


def test_epilogue_variants_select_no_accumulators_at_run_time(library):  # noqa: F811
    fsel = {}
    for name, instrs in sass_functions(library).items():
        fsel[_width(name)] = sum(1 for _, s in instrs if re.search(r"\bFSEL\b", s))
    assert len(fsel) == 12
    for pair in (False, True):
        base_bn = 128 if pair else 64
        base = fsel[(base_bn, pair)]
        for (bn, p), n in fsel.items():
            if p == pair:
                assert n - base <= 16 * (bn - base_bn) // 32, f"BN {bn} pair {pair}: {n} FSEL vs {base} at BN {base_bn}"
