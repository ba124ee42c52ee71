"""Return codes of every host-pointer entry point on the argument checks that run before any data is read: an empty batch, a NULL
required pointer, a negative batch and one instance beyond the context's capacity. No kernel runs on these paths."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HB_OK, HB_EINVAL, HB_ECAP = 0, -1, -4
MAX_BATCH = 2

# Arguments after (ctx, B): "P" a required pointer, "o" a nullable one, an int or a float a scalar of that C type.
# The last field is the code for B = max_batch + 1, or None where the call reads its inputs before it would reject the batch.
CALLS = [
    ("hb_wbc_qp_batch", [6, 4, "P", "P", "P", "P", "P", "P", "o", "o"], None),
    ("hb_wbc_solve_batch", ["P", "P", "P", "P", "o", "P", "o"], HB_ECAP),
    ("hb_wbc_assemble_batch", ["P", "P", "P", "P", "o", "P", "P", "P", "P", "P", "P"], HB_ECAP),
    ("hb_hoqp_solve_batch", ["P", "P", "o", "o"], HB_ECAP),
    ("hb_hierarchical_wbc_solve_batch", ["P", "P", "P", "P", "P", "o"], HB_ECAP),
    ("hb_hierarchical_wbc_tasks_batch", ["P", "P", "P", "P", "P"], HB_ECAP),
    ("hb_mpc_cold_start_batch", ["P", "P", "P", "P"], HB_ECAP),
    ("hb_mpc_solve_batch", ["P", "P", "P", "P", "P", "P", "o"], HB_ECAP),
    ("hb_control_step_batch", [0.002, "P", "P", "P", "P", "P", "P", "P", "o", "o", "o", "o"], HB_ECAP),
    ("hb_joint_command_batch", ["P", 0.002, "P", "P", "P", "P", "P", "o", "o", "P", "P"], HB_ECAP),
    ("hb_resident_cycle_batch", [1, 0.002, "P", "P", "P", "P", "o", "o", "o", "o"], HB_ECAP),
    ("hb_resident_read_batch", ["o", "o", "o"], HB_EINVAL),
    ("hb_resident_write_batch", ["P", "P", "P", "o", "o", "o"], HB_ECAP),
    ("hb_resident_read_grid_batch", ["P", "P"], HB_EINVAL),
    ("hb_time_grid_batch", ["P", "P", "P", "P", "o"], HB_ECAP),
    ("hb_reference_expand_grid_batch", ["P", "P", "P", "P", "P"], HB_ECAP),
    ("hb_mpc_solve_grid_batch", ["P", "P", "P", "P", "P", "P", "P", "P", "o"], HB_ECAP),
    ("hb_plan_references_gpu", ["P", "P", "P", "o"], HB_ECAP),
    ("hb_resident_plan_cycle_batch", [1, 0.002, "P", "P", "o", "o", "o", "o", "o"], HB_ECAP),
    ("hb_estimator_update_batch", ["P", 0.002, "P", "P", "P", "P", "P", "P", "P", "P"], HB_ECAP),
    ("hb_contact_force_estimate_batch", [250.0, 0.002, "P", "P", "P", "P", "o"], HB_ECAP),
    ("hb_actuation_batch", [0.009, "P", "P", "P", "P", "P"], HB_ECAP),
    ("hb_sim_step_batch", ["P", "P", "P", "o", "o"], HB_ECAP),
    ("hb_resident_wbc_batch", ["P", "P", "o", "P", "P", "P", "P", "o", "o"], HB_ECAP),
    ("hb_rbd_to_centroidal_batch", ["P", "P"], HB_ECAP),
    ("hb_reference_expand_batch", ["P", "P", "P", "P", "P"], HB_ECAP),
    ("hb_probe_flow_map", ["P", "P", "P", "P", "P", "o"], HB_ECAP),
    ("hb_contact_positions_batch", ["P", "P"], HB_ECAP),
]


@pytest.fixture(scope="module")
def small_ctx():
    import hunter_bipedal_control_b200 as hb
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=MAX_BATCH, device=0)
    yield ctx
    ctx.close()


def _call(ctx, name, spec, B, null_at=-1):
    dummy = np.zeros(1 << 12)      # large enough for every argument at B <= max_batch + 1; never read on these paths
    args = []
    for k, a in enumerate(spec):
        if isinstance(a, str):
            args.append(None if k == null_at else C.c_void_p(dummy.ctypes.data))
        elif isinstance(a, float):
            args.append(C.c_double(a))
        else:
            args.append(C.c_int(a))
    return getattr(ctx._lib, name)(ctx._h, C.c_int(B), *args)


def test_every_host_pointer_entry_point_is_listed():
    from hunter_bipedal_control_b200 import EXPORTED_SYMBOLS
    host = {s for s in EXPORTED_SYMBOLS if s.startswith("hb_") and not s.endswith("_dev") and s not in (
        "hb_default_config", "hb_create", "hb_destroy", "hb_sync", "hb_strerror", "hb_last_cuda_error", "hb_launch_count", "hb_last_reference_upload_bytes",
        "hb_stream", "hb_profile_enable", "hb_profile_read") and not s.startswith("hb_shard_")}
    listed = {c[0] for c in CALLS}
    assert listed <= host
    with_ctx = {s for s in host if s.endswith(("_batch", "_gpu")) or s == "hb_probe_flow_map"}
    assert with_ctx == listed, sorted(with_ctx ^ listed)


@pytest.mark.parametrize("name,spec,over_cap", CALLS, ids=[c[0] for c in CALLS])
def test_host_pointer_return_codes(small_ctx, name, spec, over_cap):
    c0 = small_ctx.launch_count
    assert _call(small_ctx, name, spec, 0) == HB_OK
    assert _call(small_ctx, name, spec, -1) == HB_EINVAL
    for k, a in enumerate(spec):
        if a == "P":
            assert _call(small_ctx, name, spec, 1, null_at=k) == HB_EINVAL, k
    if over_cap is not None:
        assert _call(small_ctx, name, spec, MAX_BATCH + 1) == over_cap
    assert small_ctx.launch_count == c0
