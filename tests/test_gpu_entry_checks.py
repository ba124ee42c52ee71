"""Argument checks of the entry points that take (ctx, B), on paths that run no kernel: the device-pointer forms' return codes on an empty
batch, a negative batch, a NULL required pointer and one instance beyond capacity; the scalar parameters both forms reject; and a NaN
actuation delay, which both actuation forms reject like the rollout does."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HB_OK, HB_EINVAL, HB_ECAP = 0, -1, -4
MAX_BATCH = 2
NAN = float("nan")

# Arguments after (ctx, B): "P" a required pointer, "o" a nullable one, "sim" a required pointer to valid hb_sim_params (the device form
# reads it before the empty-batch test), a ctypes scalar as is. The last field says whether the form rejects B > max_batch (HB_ECAP).
DEV_CALLS = [
    ("hb_wbc_qp_batch_dev", [C.c_int(6), C.c_int(4), "P", "P", "P", "P", "P", "P", "o", "o"], False),
    ("hb_wbc_qp_rows_batch_dev", [C.c_int(6), C.c_int(4), "P", "P", "P", "P", "P", "P", "P", "o", "o"], False),
    ("hb_wbc_solve_batch_dev", ["P", "P", "P", "P", "o", "P", "o"], True),
    ("hb_wbc_assemble_batch_dev", ["P", "P", "P", "P", "o", "P", "P", "P", "P", "P", "P"], False),
    ("hb_hoqp_solve_batch_dev", ["P", "P", "o", "o"], True),
    ("hb_hierarchical_wbc_solve_batch_dev", ["P", "P", "P", "P", "P", "o"], True),
    ("hb_mpc_cold_start_batch_dev", ["P", "P", "P", "P"], False),
    ("hb_mpc_solve_batch_dev", ["P", "P", "P", "P", "P", "P", "o"], True),
    ("hb_mpc_solve_grid_batch_dev", ["P", "P", "P", "P", "P", "P", "P", "P", "o"], True),
    ("hb_policy_eval_batch_dev", [C.c_double(0.002), "P", "P", "P", "P", "P", "o"], False),
    ("hb_policy_eval_grid_batch_dev", [C.c_double(0.002), "P", "P", "P", "P", "P", "P", "P", "o"], False),
    ("hb_time_grid_batch_dev", ["P", "P", "P", "P", "o"], False),
    ("hb_reference_expand_batch_dev", ["P", "P", "P", "P", "P"], False),
    ("hb_reference_expand_grid_batch_dev", ["P", "P", "P", "P", "P"], False),
    ("hb_control_step_batch_dev", [C.c_double(0.002), "P", "P", "P", "P", "P", "P", "P", "o", "P", "o", "o"], True),
    ("hb_resident_cycle_batch_dev", [C.c_int(1), C.c_double(0.002), "P", "P", "P", "P", "o", "P", "o", "o"], True),
    ("hb_resident_wbc_batch_dev", ["P", "P", "o", "P", "P", "P", "P", "o", "o"], False),
    ("hb_plan_references_batch_dev", ["P", "o", "P", "P", "o"], False),
    ("hb_estimator_update_batch_dev", ["P", C.c_double(0.002), "P", "P", "P", "P", "P", "P", "P", "P"], False),
    ("hb_sim_read_sensors_batch_dev", ["P", C.c_int64(0), C.c_double(0.002), "P", "P", "P", "P", "P", "P", "P"], True),
    ("hb_contact_force_estimate_batch_dev", [C.c_double(250.0), C.c_double(0.002), "P", "P", "P", "P", "o"], False),
    ("hb_actuation_batch_dev", [C.c_double(0.009), "P", "P", "P", "P", "P"], False),
    ("hb_sim_step_batch_dev", ["sim", "P", "P", "o", "o"], False),
    ("hb_joint_command_batch_dev", ["P", C.c_double(0.002), "P", "P", "P", "P", "P", "o", "o", "P", "P"], False),
    ("hb_rbd_to_centroidal_batch_dev", ["P", "P"], False),
    ("hb_contact_positions_batch_dev", ["P", "P"], False),
    ("hb_probe_flow_map_dev", ["P", "P", "P", "P", "P", "o"], False),
]
# covered with real episodes by test_gpu_rollout_episodes.py and test_gpu_rollout_estimation.py
ROLLOUTS = {"hb_rollout_batch_dev", "hb_rollout_estimated_batch_dev"}


@pytest.fixture(scope="module")
def small_ctx():
    import hunter_bipedal_control_b200 as hb
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=MAX_BATCH, device=0)
    yield ctx
    ctx.close()


def _call(ctx, name, spec, B, null_at=-1):
    import hunter_bipedal_control_b200 as hb
    dummy = np.zeros(1 << 12)      # host memory, never read: every call here is rejected before a kernel could see it
    sim = hb.default_sim_params()
    args = []
    for k, a in enumerate(spec):
        if k == null_at:
            args.append(None)
        elif a == "sim":
            args.append(C.byref(sim))
        elif isinstance(a, str):
            args.append(C.c_void_p(dummy.ctypes.data))
        else:
            args.append(a)
    return getattr(ctx._lib, name)(ctx._h, C.c_int(B), *args)


def test_every_device_pointer_entry_point_is_listed():
    from hunter_bipedal_control_b200 import EXPORTED_SYMBOLS
    dev = {s for s in EXPORTED_SYMBOLS if s.startswith("hb_") and s.endswith("_dev") and not s.startswith("hb_shard_")}
    listed = {c[0] for c in DEV_CALLS}
    assert listed <= dev and not listed & ROLLOUTS
    assert dev - ROLLOUTS == listed, sorted((dev - ROLLOUTS) ^ listed)


@pytest.mark.parametrize("name,spec,capped", DEV_CALLS, ids=[c[0] for c in DEV_CALLS])
def test_device_pointer_return_codes(small_ctx, name, spec, capped):
    c0 = small_ctx.launch_count
    assert _call(small_ctx, name, spec, 0) == HB_OK
    assert _call(small_ctx, name, spec, -1) == HB_EINVAL
    for k, a in enumerate(spec):
        if a in ("P", "sim"):
            assert _call(small_ctx, name, spec, 1, null_at=k) == HB_EINVAL, k
    if capped:
        assert _call(small_ctx, name, spec, MAX_BATCH + 1) == HB_ECAP
    assert small_ctx.launch_count == c0


def _sim_params(**kw):
    import hunter_bipedal_control_b200 as hb
    p = hb.default_sim_params()
    for k, v in kw.items():
        setattr(p, k, v)
    return C.byref(p)


def _noise(**kw):
    import hunter_bipedal_control_b200 as hb
    n = hb.HbSensorNoise()
    for k, v in kw.items():
        setattr(n, k, v)
    return C.byref(n)


# Codes at B = 0, 1, max_batch + 1. A device form checks its scalars with its pointers, before the batch. A host form checks them
# where it checked them before staging: after the capacity check (AFTER_CAP), with the pointers (FIRST), or, for the QP shape of a form
# without a capacity check, after the empty-batch test (UNCAPPED).
FIRST = (HB_EINVAL, HB_EINVAL, HB_EINVAL)
AFTER_CAP = (HB_OK, HB_EINVAL, HB_ECAP)
UNCAPPED = (HB_OK, HB_EINVAL, HB_EINVAL)

# (id, host form or None, its codes, device form, its codes, arguments after (ctx, B) with "P" a dummy pointer and "o" a NULL one)
SCALAR_CASES = []
for kw in (dict(dt=0.0), dict(dt=-0.002), dict(dt=NAN), dict(substeps=0), dict(substeps=1001)):
    SCALAR_CASES.append(("sim_" + "_".join("%s=%s" % i for i in kw.items()), "hb_sim_step_batch", AFTER_CAP, "hb_sim_step_batch_dev", FIRST,
                         lambda kw=kw: [_sim_params(**kw), "P", "P", "o", "o"]))
SCALAR_CASES.append(("delay=-1", "hb_actuation_batch", AFTER_CAP, "hb_actuation_batch_dev", FIRST,
                     lambda: [C.c_double(-1.0), "P", "P", "P", "P", "P"]))
for cutoff, dt in ((0.0, 0.002), (250.0, 0.0)):
    SCALAR_CASES.append(("cutoff=%g_dt=%g" % (cutoff, dt), "hb_contact_force_estimate_batch", AFTER_CAP, "hb_contact_force_estimate_batch_dev", FIRST,
                         lambda cutoff=cutoff, dt=dt: [C.c_double(cutoff), C.c_double(dt), "P", "P", "P", "P", "o"]))
for tag, noise, tick, accel_dt in (("sigma=-0.1", dict(orientation=-0.1), 0, 0.002), ("sigma=nan", dict(joint_velocity=NAN), 0, 0.002),
                                   ("tick=-1", {}, -1, 0.002), ("accel_dt=0", {}, 0, 0.0)):
    SCALAR_CASES.append(("sensors_" + tag, "hb_sim_read_sensors", FIRST, "hb_sim_read_sensors_batch_dev", FIRST,
                         lambda noise=noise, tick=tick, accel_dt=accel_dt: [_noise(**noise), C.c_int64(tick), C.c_double(accel_dt)] + ["P"] * 7))
for n, m in ((0, 4), (81, 4), (6, 161)):       # n = 0, n > QP_MAX_N, m > QP_MAX_M
    SCALAR_CASES.append(("qp_n=%d_m=%d" % (n, m), "hb_wbc_qp_batch", UNCAPPED, "hb_wbc_qp_batch_dev", UNCAPPED,
                         lambda n=n, m=m: [C.c_int(n), C.c_int(m)] + ["P"] * 6 + ["o", "o"]))
    SCALAR_CASES.append(("qp_rows_n=%d_m=%d" % (n, m), None, None, "hb_wbc_qp_rows_batch_dev", UNCAPPED,
                         lambda n=n, m=m: [C.c_int(n), C.c_int(m)] + ["P"] * 7 + ["o", "o"]))


def _call_args(ctx, name, B, args):
    dummy = np.zeros(1 << 12)      # host memory, never read: an invalid scalar rejects every call before a kernel could see it
    conv = [C.c_void_p(dummy.ctypes.data) if a == "P" else (None if a == "o" else a) for a in args]
    return getattr(ctx._lib, name)(ctx._h, C.c_int(B), *conv)


@pytest.mark.parametrize("case", SCALAR_CASES, ids=[c[0] for c in SCALAR_CASES])
def test_scalar_rejections(small_ctx, case):
    _, host, host_codes, dev, dev_codes, make_args = case
    c0 = small_ctx.launch_count
    for k, B in enumerate((0, 1, MAX_BATCH + 1)):
        assert _call_args(small_ctx, dev, B, make_args()) == dev_codes[k], (dev, B)
        if host:
            assert _call_args(small_ctx, host, B, make_args()) == host_codes[k], (host, B)
    assert small_ctx.launch_count == c0


def test_nan_delay_is_rejected_by_both_actuation_forms(small_ctx):
    import torch

    import hunter_bipedal_control_b200 as hb
    c0 = small_ctx.launch_count
    time, command, rbd, tau = np.zeros(1), np.zeros((1, 50)), np.zeros((1, 32)), np.zeros((1, 10))
    state = hb.actuation_states(1)
    lib, h = small_ctx._lib, small_ctx._h
    p = lambda a: C.c_void_p(a.ctypes.data)      # noqa: E731
    assert lib.hb_actuation_batch(h, 1, C.c_double(NAN), p(time), state, p(command), p(rbd), p(tau)) == HB_EINVAL
    dev = torch.device("cuda", 0)
    d_time, d_cmd, d_rbd, d_tau = (torch.zeros(s, dtype=torch.float64, device=dev) for s in ((1,), (1, 50), (1, 32), (1, 10)))
    d_state = torch.zeros(C.sizeof(hb.HbActuationState), dtype=torch.uint8, device=dev)
    q = lambda t: C.c_void_p(t.data_ptr())       # noqa: E731
    assert lib.hb_actuation_batch_dev(h, 1, C.c_double(NAN), q(d_time), q(d_state), q(d_cmd), q(d_rbd), q(d_tau)) == HB_EINVAL
    torch.cuda.synchronize()
    assert small_ctx.launch_count == c0
