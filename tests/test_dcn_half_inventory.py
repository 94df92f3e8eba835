"""CPU: the half-precision DCN kernel instantiations compiled into the library are exactly
test_dcn_half_gpu.HALF_VARIANTS, and each of them is expected to run by at least one GPU case."""
import re
import shutil

import pytest

from tests import test_dcn_half_gpu
from tests.test_kernel_inventory import so_path  # noqa: F401  (fixture)
from tests import wgmma_variants as wv


def compiled_half_variants(so):
    import subprocess
    dump = subprocess.run([shutil.which("cuobjdump"), "-symbols", so], check=True, capture_output=True, text=True).stdout
    mangled = sorted(set(re.findall(r"\b_Z\w+", dump)))
    names = subprocess.run([shutil.which("cu++filt")], input="\n".join(mangled), check=True, capture_output=True,
                           text=True).stdout.splitlines()
    return {n for n in map(wv.normalise, names) if re.fullmatch(r"dcn_(fwd|wgrad|dgrad)_half_kernel<\w+>", n)}


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None,
                    reason="needs cuobjdump and cu++filt from the CUDA toolkit")
def test_compiled_half_instantiations_are_known(so_path):  # noqa: F811
    found = compiled_half_variants(so_path)
    assert found == test_dcn_half_gpu.HALF_VARIANTS, ("unknown: %s; not compiled: %s"
                                                      % (sorted(found - test_dcn_half_gpu.HALF_VARIANTS),
                                                         sorted(test_dcn_half_gpu.HALF_VARIANTS - found)))


def test_every_half_variant_has_a_gpu_case():
    assert test_dcn_half_gpu.VARIANTS == test_dcn_half_gpu.HALF_VARIANTS
