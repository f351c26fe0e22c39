"""Record the reference's answers for the tests that need a GPU (tests/refreplay.py), without one.

    ACB_RECORD_REFERENCE=1 python -m pytest tests -m "not gpu"     # the CPU tests record their own entries
    python tests/golden/record_reference.py                         # then these

Needs the unmodified reference extension in oracle/_ref (`make -C oracle ref`).  What the reference answers does not
depend on the device the drop-in searches on, so the gpu tests' questions are asked here with the drop-in on the
CPU emulation of the kernels (tests/emul.py), and the digests of the full-size comparisons are computed from the
same seeded workloads the tests build.
"""
import os
import sys

os.environ["ACB_RECORD_REFERENCE"] = "1"
TESTS = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.dirname(TESTS), TESTS]

import pytest  # noqa: E402

import emul  # noqa: E402
import test_gpu_parity as gp  # noqa: E402
import test_iter_long_set as ils  # noqa: E402
import test_search_args_differential as sad  # noqa: E402
from pyahocorasick_b200 import synth  # noqa: E402


def as_test(tid, fn, *args):
    os.environ["PYTEST_CURRENT_TEST"] = f"tests/{tid} (call)"
    mp = pytest.MonkeyPatch()
    try:
        emul.install(mp, "filter")
        fn(*args)
    finally:
        mp.undo()


def main():
    for fl in ("bytes", "unicode"):
        as_test(f"test_iter_long_set.py::test_iter_long_set_matches_the_reference_on_gpu[{fl}]",
                ils.test_iter_long_set_matches_the_reference_on_gpu, fl)
    as_test("test_iter_long_set.py::test_iter_long_long_stream_on_gpu", ils.test_iter_long_long_stream_on_gpu)
    for name in ("iter_ranges_and_white_space", "find_all_ranges", "batch_input_forms_equal_looping_the_reference",
                 "key_sequences_iter_and_iter_long", "searches_between_random_mutations", "iter_long_ranges_and_batch"):
        for fl in ("bytes", "unicode"):
            as_test(f"test_search_args_differential.py::test_{name}_on_gpu[{fl}]", getattr(sad, f"test_{name}_on_gpu"), fl)
    for fl in ("bytes", "unicode"):
        for ws in (False, True):
            as_test(f"test_search_args_differential.py::test_iter_set_at_random_points_on_gpu[{fl}-{ws}]",
                    sad.test_iter_set_at_random_points_on_gpu, fl, ws)
    gp.reference_c2_sample()
    for name, make in (("c2_rows", lambda: synth.make("C2", scale=1.0)), ("c3_rows", lambda: synth.make("C3", scale=1.0)),
                       ("c4_rows", gp.c4_with_straddlers), ("c5_rows", lambda: synth.make("C5", scale=0.125))):
        w = make()
        print(name, gp.reference_rows(name, w, gp.FULL_ROWS[name](w)), flush=True)
        del w


if __name__ == "__main__":
    main()
