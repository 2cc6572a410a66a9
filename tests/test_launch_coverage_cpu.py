"""Every prims function a census workload calls is checked element by element somewhere: it is claimed by exactly one launch
census (GEMM, attention, norm, glue, optimizer; each has a float64 check of every recorded launch) or by ALLOWLIST, which names the test
that covers it and why it sits outside a census.  A new kernel that the training steps launch without a check fails here.
The workloads are those of tests/golden/make_glue_launches.py (a superset of the other kernel censuses' workloads) and of
tests/golden/make_optim_launches.py (the optimizer steps, the stable-LoRA pass and the gradient compression), run once on the
meta device with every public prims function wrapped by a recorder."""
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_attn_launches as MA   # noqa: E402
import make_glue_launches as MG   # noqa: E402
import make_norm_launches as MN   # noqa: E402
import make_optim_launches as MO   # noqa: E402

CENSUSES = {
    "gemm": ("conv_fwd", "conv_dgrad", "conv_wgrad", "bgemm"),                       # tests/test_gemm_step_gpu.py
    "attention": tuple(k for k in MA.KINDS if k != "composite") + ("softmax_fwd", "softmax_bwd"),   # tests/test_attn_step_gpu.py
    "norm": MN.KINDS,                                                                  # tests/test_norm_step_gpu.py
    "glue": MG.KINDS,                                                                  # tests/test_glue_step_gpu.py
    "optimizer": MO.KINDS,                                                             # tests/test_optim_step_gpu.py
}
ALLOWLIST = {
    "out_hw": "host helper: no kernel",
    "stats_alloc": "host helper: a zeroed buffer, no kernel",
}


def claims():
    """{prims function: [claimants]} over the censuses and the allowlist."""
    out = {}
    for census, names in CENSUSES.items():
        for n in names:
            out.setdefault(n, []).append(census)
    for n in ALLOWLIST:
        out.setdefault(n, []).append("allowlist")
    return out


_CALLED = []


def called():
    """The prims functions the census workloads call, recorded once."""
    if not _CALLED:
        seen = set()

        def observe(name, fn):
            def run(*args, **kw):
                seen.add(name)
                return fn(*args, **kw)
            return run

        MG.run_workloads(observe=observe)
        MO.run_workloads(observe=observe)
        _CALLED.append(sorted(seen))
    return _CALLED[0]


def unclaimed(names, table):
    """The functions of `names` that `table` does not claim exactly once, with their claimants."""
    return {n: table.get(n, []) for n in names if len(table.get(n, [])) != 1}


def test_every_called_prim_is_claimed_once():
    bad = unclaimed(called(), claims())
    assert not bad, f"prims functions the steps call without exactly one float64 check (census or allowlist): {bad}"


def test_claims_name_prims_functions():
    from t2v_b200 import prims
    missing = sorted(n for n in claims() if not callable(getattr(prims, n, None)))
    assert not missing, missing


@pytest.mark.parametrize("census", list(CENSUSES))
def test_removing_a_kind_fails(census):
    """Dropping one called function from a census leaves it unclaimed."""
    names = [n for n in CENSUSES[census] if n in called()]
    assert names, f"the workloads call nothing of the {census} census"
    table = claims()
    table[names[0]] = [c for c in table[names[0]] if c != census]
    assert names[0] in unclaimed(called(), table)
