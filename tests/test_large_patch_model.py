"""CPU: the host model of patch_large_kernel's chunked arrival sweep (tests/large_patch_model.py) against the oracle's
applyChange return values and the host closed forms (peritext_b200/patches.py), on the corner, adversarial and multi-trip
catalogues of tests/test_gpu_patch_bounds.py, at chunk sizes from one op to more than a whole log."""
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.packing import _root_text_list
from tests.large_patch_model import sweep_patches
from tests.test_gpu_patch_bounds import adversarial_cases, corner_cases, list_ops, trip_cases
from tests.test_patch_closed_form import closed_form_patches

CATALOGUES = {"corners": corner_cases, "adversarial": adversarial_cases, "trips": trip_cases}


@pytest.mark.parametrize("B", [1, 2, 32, 1024])
@pytest.mark.parametrize("group", list(CATALOGUES))
def test_sweep_model_equals_the_oracle_and_the_closed_forms(group, B):
    for c in CATALOGUES[group]():
        fresh = O("observer")
        want = []
        for ch in c.changes:
            want += [p for p in fresh.applyChange(ch) if p["action"] != "makeList"]
        elements = fresh.elements()
        pos = {e["elemId"]: k for k, e in enumerate(elements)}
        got = [p for ps in sweep_patches(list_ops(c.changes), pos, B) for p in ps]
        assert got == want, (c.name, B)
        assert got == closed_form_patches(c.changes, elements, _root_text_list(c.changes)), (c.name, B)
