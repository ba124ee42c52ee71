#!/usr/bin/env python3
"""Generate include/hunter_model_constants.h from the reference's URDF and INFO files.

Usage: gen_model.py REFERENCE_CHECKOUT [OUT]. The generated header is committed, so nothing at run time needs the
reference tree; tests/golden/hunter_config/ holds the three source files for the regeneration test.

Sources (relative to the reference checkout):
  legged_examples/legged_hunter/legged_hunter_description/urdf/hunter.urdf   (tree, inertias, limits)
  legged_controllers/config/hunter/task.info                                 (weights, gains)
  legged_controllers/config/hunter/reference.info                            (default joints, gaits)
Fixed-joint children (imu_link, the four contact links) are merged into their parent body the way
a URDF parser with fixed-joint reduction does (Pinocchio's buildModel, used by the reference through
legged_interface/src/LeggedInterface.cpp:188-200).
"""
import sys, re, os
import xml.etree.ElementTree as ET
import numpy as np

if len(sys.argv) < 2:
    sys.exit(__doc__)
REF = sys.argv[1]
URDF = os.path.join(REF, "legged_examples/legged_hunter/legged_hunter_description/urdf/hunter.urdf")
TASK = os.path.join(REF, "legged_controllers/config/hunter/task.info")
REFI = os.path.join(REF, "legged_controllers/config/hunter/reference.info")
OUT = sys.argv[2] if len(sys.argv) > 2 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "hunter_model_constants.h")

JOINTS = ["leg_l1_joint", "leg_l2_joint", "leg_l3_joint", "leg_l4_joint", "leg_l5_joint",
          "leg_r1_joint", "leg_r2_joint", "leg_r3_joint", "leg_r4_joint", "leg_r5_joint"]  # ModelSettings.h:59-60
CONTACTS = ["leg_l_f1_link", "leg_r_f1_link", "leg_l_f2_link", "leg_r_f2_link"]          # ModelSettings.h:62


def vec(s, n=3):
    return np.array([float(x) for x in s.split()]) if s is not None else np.zeros(n)


def rpy_to_R(rpy):
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def parse():
    root = ET.parse(URDF).getroot()
    links = {}
    for l in root.findall("link"):
        i = l.find("inertial")
        if i is None:
            links[l.get("name")] = dict(m=0.0, c=np.zeros(3), I=np.zeros((3, 3)))
            continue
        o = i.find("origin")
        xyz = vec(o.get("xyz")) if o is not None else np.zeros(3)
        rpy = vec(o.get("rpy")) if (o is not None and o.get("rpy")) else np.zeros(3)
        m = float(i.find("mass").get("value"))
        it = i.find("inertia")
        g = lambda k: float(it.get(k))
        I = np.array([[g("ixx"), g("ixy"), g("ixz")], [g("ixy"), g("iyy"), g("iyz")], [g("ixz"), g("iyz"), g("izz")]])
        R = rpy_to_R(rpy)
        links[l.get("name")] = dict(m=m, c=xyz, I=R @ I @ R.T)
    joints = {}
    for j in root.findall("joint"):
        o = j.find("origin")
        a = j.find("axis")
        lim = j.find("limit")
        joints[j.get("name")] = dict(
            type=j.get("type"), parent=j.find("parent").get("link"), child=j.find("child").get("link"),
            xyz=vec(o.get("xyz")) if o is not None else np.zeros(3),
            rpy=vec(o.get("rpy")) if (o is not None and o.get("rpy")) else np.zeros(3),
            axis=vec(a.get("xyz")) if a is not None else None,
            lim=(float(lim.get("lower")), float(lim.get("upper")), float(lim.get("effort")), float(lim.get("velocity")))
            if lim is not None else None)
    return links, joints


def merge(body, add_m, add_c, add_I):
    """Merge a rigidly attached inertia (mass add_m, com add_c in body frame, inertia about its com)."""
    m0, c0, I0 = body["m"], body["c"], body["I"]
    m = m0 + add_m
    if m == 0:
        return
    c = (m0 * c0 + add_m * add_c) / m
    def shift(I, mm, d):  # parallel axis: inertia about point displaced by d from the com
        return I + mm * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
    I = shift(I0, m0, c0 - c) + shift(add_I, add_m, add_c - c)
    body["m"], body["c"], body["I"] = m, c, I


def info_block(text, name):
    m = re.search(r"^\s*" + re.escape(name) + r"\s*\{", text, re.M)
    assert m, name
    i = m.end(); depth = 1; j = i
    while depth:
        ch = text[j]
        depth += ch == "{"; depth -= ch == "}"; j += 1
    return text[i:j - 1]


def info_matrix_entries(block):
    out = {}
    for m in re.finditer(r"\((\d+),\s*(\d+)\)\s+([-+0-9.eE]+)", block):
        out[(int(m.group(1)), int(m.group(2)))] = float(m.group(3))
    return out


def info_scalar(block, key):
    m = re.search(r"^\s*" + re.escape(key) + r"\s+([-+0-9.eE]+)", block, re.M)
    assert m, key
    return float(m.group(1))


def strip_comments(t):
    return "\n".join(l.split(";")[0] if not re.match(r"^\s*\(", l) else l.split(";")[0] for l in t.splitlines())


def main():
    links, joints = parse()
    # --- bodies: 0 = base, 1..10 = moving links in JOINTS order
    bodies = [dict(name="base_link", parent=-1, xyz=np.zeros(3), axis=np.zeros(3), **links["base_link"])]
    body_of_link = {"base_link": 0}
    for jn in JOINTS:
        j = joints[jn]
        assert j["type"] == "revolute" and np.allclose(j["rpy"], 0), jn
        assert abs(np.abs(j["axis"]).sum() - 1) < 1e-12 and np.abs(j["axis"]).max() == 1, "axis must be a signed unit axis"
        b = dict(name=j["child"], parent=body_of_link[j["parent"]], xyz=j["xyz"], axis=j["axis"], lim=j["lim"],
                 **links[j["child"]])
        body_of_link[j["child"]] = len(bodies)
        bodies.append(b)
    # --- fixed joints: merge child into parent, remember frame offsets
    frames = {}
    for jn, j in joints.items():
        if j["type"] != "fixed":
            continue
        assert np.allclose(j["rpy"], 0), jn
        pb = body_of_link[j["parent"]]
        ch = links[j["child"]]
        merge(bodies[pb], ch["m"], j["xyz"] + ch["c"], ch["I"])
        frames[j["child"]] = (pb, j["xyz"])
        body_of_link[j["child"]] = pb
    total_mass = sum(b["m"] for b in bodies)

    task = open(TASK).read()
    refi = open(REFI).read()
    ts, rs = strip_comments(task), strip_comments(refi)

    Q = info_matrix_entries(info_block(ts, "Q"))
    Qs = info_scalar(info_block(ts, "Q"), "scaling")
    R = info_matrix_entries(info_block(ts, "R"))
    Rs = info_scalar(info_block(ts, "R"), "scaling")
    x0 = info_matrix_entries(info_block(ts, "initialState"))
    dj = info_matrix_entries(info_block(rs, "defaultJointState"))
    tl = info_matrix_entries(info_block(ts, "torqueLimitsTask"))

    def arr(name, vals, fmt="%.17g"):
        return "static const double %s[%d] = {%s};\n" % (name, len(vals), ", ".join(fmt % v for v in vals))

    o = []
    o.append("/* GENERATED by tools/gen_model.py from the reference's hunter.urdf / task.info / reference.info.\n"
             " * Do not edit. Data only (no algorithm): shared by the CUDA product path and the CPU oracle.\n"
             " * Bodies: 0 = base_link (+imu_link), 1..5 = leg_l1..l5 (+toe/heel links in l5), 6..10 = leg_r1..r5.\n"
             " * Citations: urdf/hunter.urdf (joints :88-228,:416-556; contact frames :253-294,:581-622),\n"
             " * legged_controllers/config/hunter/task.info, reference.info. */\n")
    o.append("#ifndef HUNTER_MODEL_CONSTANTS_H\n#define HUNTER_MODEL_CONSTANTS_H\n\n")
    o.append("#define HB_NBODY 11\n#define HB_NJ 10\n#define HB_NQ 16\n#define HB_NX 22\n#define HB_NU 22\n#define HB_NC 4\n#define HB_NWBC 38\n\n")
    o.append("static const int HB_PARENT[11] = {%s};\n" % ", ".join(str(b["parent"]) for b in bodies))
    o.append(arr("HB_JOINT_XYZ", [v for b in bodies for v in b["xyz"]]).replace("[33]", "[11*3]"))
    o.append(arr("HB_JOINT_AXIS", [v for b in bodies for v in b["axis"]]).replace("[33]", "[11*3]"))
    o.append(arr("HB_BODY_MASS", [b["m"] for b in bodies]))
    o.append(arr("HB_BODY_COM", [v for b in bodies for v in b["c"]]).replace("[33]", "[11*3]"))
    o.append(arr("HB_BODY_INERTIA", [v for b in bodies for v in b["I"].reshape(-1)]).replace("[99]", "[11*9]"))
    o.append("#define HB_TOTAL_MASS %.17g\n" % total_mass)
    o.append("static const int HB_CONTACT_BODY[4] = {%s};\n" % ", ".join(str(frames[c][0]) for c in CONTACTS))
    o.append(arr("HB_CONTACT_OFFSET", [v for c in CONTACTS for v in frames[c][1]]).replace("[12]", "[4*3]"))
    o.append(arr("HB_JOINT_LOWER", [b["lim"][0] for b in bodies[1:]]))
    o.append(arr("HB_JOINT_UPPER", [b["lim"][1] for b in bodies[1:]]))
    o.append(arr("HB_JOINT_VEL_LIMIT", [b["lim"][3] for b in bodies[1:]]))
    o.append("\n/* task.info */\n")
    o.append(arr("HB_Q_DIAG", [Q[(i, i)] * Qs for i in range(22)]))
    o.append(arr("HB_R_TASKSPACE_DIAG", [R[(i, i)] * Rs for i in range(24)]))
    o.append(arr("HB_INITIAL_STATE", [x0[(i, 0)] for i in range(22)]))
    o.append(arr("HB_DEFAULT_JOINT_STATE", [dj[(i, 0)] for i in range(10)]))
    o.append(arr("HB_WBC_TORQUE_LIMITS", [tl[(i, 0)] for i in range(5)]))
    scal = [
        ("HB_GRAVITY", 9.81),
        ("HB_POSITION_ERROR_GAIN", info_scalar(info_block(ts, "model_settings"), "positionErrorGain")),
        ("HB_PHASE_TRANSITION_STANCE_TIME", info_scalar(info_block(ts, "model_settings"), "phaseTransitionStanceTime")),
        ("HB_FRICTION_MU", info_scalar(info_block(ts, "frictionConeSoftConstraint"), "frictionCoefficient")),
        ("HB_FRICTION_BARRIER_MU", info_scalar(info_block(ts, "frictionConeSoftConstraint"), "mu")),
        ("HB_FRICTION_BARRIER_DELTA", info_scalar(info_block(ts, "frictionConeSoftConstraint"), "delta")),
        ("HB_FRICTION_REGULARIZATION", 25.0),       # FrictionConeConstraint.h:77
        ("HB_FRICTION_HESSIAN_SHIFT", 1e-6),        # FrictionConeConstraint.h:78
        ("HB_SOFT_SWING_WEIGHT", info_scalar(info_block(ts, "softSwingTraj"), "weight")),
        ("HB_XY_POSITION_GAIN", 3.0),               # LeggedRobotPreComputation.cpp:115-117
        ("HB_ZEROVEL_Z_GAIN", 3.0),                 # LeggedInterface.cpp:441-443
        ("HB_ZEROVEL_Z_OFFSET", -0.06),             # LeggedInterface.cpp:441
        ("HB_LIMIT_POS_MU", 1.0), ("HB_LIMIT_POS_DELTA", 0.1),      # LeggedInterface.cpp:336
        ("HB_LIMIT_VEL_MU", 1.0), ("HB_LIMIT_VEL_DELTA", 0.1),      # LeggedInterface.cpp:337
        ("HB_LIMIT_FORCE_MU", 0.1), ("HB_LIMIT_FORCE_DELTA", 1.0),  # LeggedInterface.cpp:338
        ("HB_LIMIT_FORCE_MAX", 350.0),                              # LeggedInterface.cpp:352
        ("HB_SQP_G_MAX", info_scalar(info_block(ts, "sqp"), "g_max")),
        ("HB_SQP_G_MIN", info_scalar(info_block(ts, "sqp"), "g_min")),
        ("HB_SQP_DELTA_TOL", info_scalar(info_block(ts, "sqp"), "deltaTol")),
        ("HB_SQP_DT", info_scalar(info_block(ts, "sqp"), "dt")),
        ("HB_MPC_TIME_HORIZON", info_scalar(info_block(ts, "mpc"), "timeHorizon")),
        ("HB_WBC_FRICTION_MU", info_scalar(info_block(ts, "frictionConeTask"), "frictionCoefficient")),
        ("HB_WBC_SWING_KP", info_scalar(info_block(ts, "swingLegTask"), "kp")),
        ("HB_WBC_SWING_KD", info_scalar(info_block(ts, "swingLegTask"), "kd")),
        ("HB_WBC_BASE_HEIGHT_KP", info_scalar(info_block(ts, "baseHeightTask"), "kp")),
        ("HB_WBC_BASE_HEIGHT_KD", info_scalar(info_block(ts, "baseHeightTask"), "kd")),
        ("HB_WBC_BASE_ANGULAR_KP", info_scalar(info_block(ts, "baseAngularTask"), "kp")),
        ("HB_WBC_BASE_ANGULAR_KD", info_scalar(info_block(ts, "baseAngularTask"), "kd")),
        ("HB_WBC_WEIGHT_SWING", info_scalar(info_block(ts, "weight"), "swingLeg")),
        ("HB_WBC_WEIGHT_BASE", info_scalar(info_block(ts, "weight"), "baseAccel")),
        ("HB_WBC_WEIGHT_FORCE", info_scalar(info_block(ts, "weight"), "contactForce")),
        ("HB_SWING_LIFTOFF_VEL", info_scalar(info_block(ts, "swing_trajectory_config"), "liftOffVelocity")),
        ("HB_SWING_TOUCHDOWN_VEL", info_scalar(info_block(ts, "swing_trajectory_config"), "touchDownVelocity")),
        ("HB_SWING_HEIGHT", info_scalar(info_block(ts, "swing_trajectory_config"), "swingHeight")),
        ("HB_SWING_TIME_SCALE", info_scalar(info_block(ts, "swing_trajectory_config"), "swingTimeScale")),
        ("HB_FEET_BIAS_X1", info_scalar(info_block(ts, "swing_trajectory_config"), "feet_bias_x1")),
        ("HB_FEET_BIAS_X2", info_scalar(info_block(ts, "swing_trajectory_config"), "feet_bias_x2")),
        ("HB_FEET_BIAS_Y", info_scalar(info_block(ts, "swing_trajectory_config"), "feet_bias_y")),
        ("HB_FEET_BIAS_Z", info_scalar(info_block(ts, "swing_trajectory_config"), "feet_bias_z")),
        ("HB_NEXT_POSITION_Z", 0.02),   # SwingTrajectoryPlanner.h:70 default (key mismatch in task.info, SURVEY App. A)
        ("HB_COM_HEIGHT", info_scalar(rs, "comHeight")),
        ("HB_TARGET_DISPLACEMENT_VELOCITY", info_scalar(rs, "targetDisplacementVelocity")),   # goal reaching time (TargetTrajectoriesPublisher.cpp:29-38)
        ("HB_TARGET_ROTATION_VELOCITY", info_scalar(rs, "targetRotationVelocity")),
    ]
    for k, v in scal:
        o.append("#define %s %.17g\n" % (k, v))
    o.append("\n#endif\n")
    with open(OUT, "w") as f:
        f.write("".join(o))
    print("wrote", os.path.normpath(OUT), "total mass", total_mass)
    for b in bodies:
        print(b["name"], b["parent"], b["xyz"], b["axis"], b["m"], b["c"])
    for c in CONTACTS:
        print(c, frames[c])


if __name__ == "__main__":
    main()
