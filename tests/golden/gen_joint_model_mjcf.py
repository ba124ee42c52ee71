#!/usr/bin/env python3
"""Generate tests/golden/joint_model_mjcf.json: the range and frictionloss of every leg joint of the reference's MJCF model
(mujoco/model/hunter/hunter.xml), in the model's joint order leg_l1 .. leg_l5, leg_r1 .. leg_r5, as the joint models' defaults
(hb_default_joint_model) are checked against them. The URDF's <limit> and <dynamics friction> are read from tests/golden/hunter_config.

Usage: gen_joint_model_mjcf.py REFERENCE_CHECKOUT
"""
import json
import os
import sys
import xml.etree.ElementTree as ET

HERE = os.path.dirname(os.path.abspath(__file__))
NAMES = ["leg_%s%d_joint" % (s, k) for s in "lr" for k in range(1, 6)]


def main(ref):
    root = ET.parse(os.path.join(ref, "mujoco", "model", "hunter", "hunter.xml")).getroot()
    joints = {j.get("name"): j for j in root.iter("joint")}
    out = {"source": "mujoco/model/hunter/hunter.xml", "joints": NAMES,
           "range": [[float(x) for x in joints[n].get("range").split()] for n in NAMES],
           "frictionloss": [float(joints[n].get("frictionloss")) for n in NAMES],
           "autolimits": (root.find("compiler") is None or root.find("compiler").get("autolimits", "true") == "true")}
    with open(os.path.join(HERE, "joint_model_mjcf.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
