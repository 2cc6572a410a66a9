"""The GEMM planner's decisions, pinned: every launch of every problem in tests/golden/gemm_plans.json (the GEMM problems of a
cfg-2 training step and of tests/test_gemm_gpu.py, at 132 and 114 SMs) must be planned exactly as recorded.  Runs on the CPU
through t2v_gemm_plan.  A change that moves plans on purpose regenerates the table with tests/golden/make_gemm_plans.py."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_gemm_plans as M  # noqa: E402


def test_plans_match_table():
    lib = M.load()
    with open(M.OUT) as f:
        records = json.load(f)
    assert len(records) > 200
    moved = []
    for rec in records:
        for sms, want in rec["plans"].items():
            got = M.query(lib, rec["problem"], rec["env"], int(sms))
            if got != want:
                moved.append((rec["problem"], rec["env"], sms, want, got))
    assert not moved, f"{len(moved)} plans moved, first: {moved[0]}"


def test_rejected_problem_is_an_error():
    from t2v_b200 import native
    lib = M.load()
    bad = M.to_struct(M.conv_problem("fwd", 1, 8, 8, 12, 64, 3, 3, 1, (1, 1, 1, 1)))   # Cin not a multiple of 8
    out = (native.GemmPlan * 4)()
    assert lib.t2v_gemm_plan(bad, 132, out, 4) < 0
    assert b"Cin" in lib.t2v_last_error()
