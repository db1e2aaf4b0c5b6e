"""Per-robot controller tuning rows (qmb200_set_robot_tuning) and the input files a handle would need to hold one row as its own values: task.info with
the row's friction coefficients and end-effector weights, and a WBC gains file with the row's gains.  The arm gains of the control law have no file: a
reference handle takes them through qmb200_set_arm_gains."""
import os
import re

import numpy as np

from qm_control_b200 import _lib

L = _lib.TUNING_LAYOUT
TASK_KEYS = {"friction_mu": ("frictionConeSoftConstraint", "frictionCoefficient"), "wbc_friction": ("frictionConeTask", "frictionCoefficient"),
             "mu_ee_pos": ("endEffector", "muPosition"), "mu_ee_ori": ("endEffector", "muOrientation"),
             "mu_final_ee_pos": ("finalEndEffector", "muPosition"), "mu_final_ee_ori": ("finalEndEffector", "muOrientation")}
GAIN_KEYS = [("kp_swing", "kp_swing"), ("kd_swing", "kd_swing"), ("base_height_kp", "baseHeightKp"), ("base_height_kd", "baseHeightKd"),
             ("kp_base_linear", "kp_base_linear"), ("kd_base_linear", "kd_base_linear"), ("kp_base_angular", "kp_base_angular"), ("kd_base_angular", "kd_base_angular")] + \
            [("kp_arm_joint", "kp_arm_joint_%d" % (i + 1), i) for i in range(6)] + [("kd_arm_joint", "kd_arm_joint_%d" % (i + 1), i) for i in range(6)] + \
            [(f, "%s_%s" % (f, a), i) for f in ("kp_ee_linear", "kd_ee_linear", "kp_ee_angular", "kd_ee_angular") for i, a in enumerate("xyz")]


def field(row, name, i=0):
    off, w = L[name]; return float(row[off + i])


def _set_block_key(text, block, key, value):
    pat = re.compile(r"(^%s\s*\{[^}]*?^\s*%s\s+)(\S+)" % (re.escape(block), re.escape(key)), re.M | re.S)
    out, n = pat.subn(lambda m: m.group(1) + repr(float(value)), text)
    assert n == 1, (block, key)
    return out


def edited_files(directory, row, tag):
    """→ (task_file, gains_file) whose values are row's (friction coefficients, end-effector weights, WBC gains)"""
    text = open(_lib.asset("qm_task.info")).read()
    for name, (block, key) in TASK_KEYS.items():
        text = _set_block_key(text, block, key, field(row, name))
    task = os.path.join(str(directory), "task_%s.info" % tag); open(task, "w").write(text)
    lines = ["wbcGains", "{"]
    for g in GAIN_KEYS:
        lines.append("  %s %r" % (g[1], field(row, g[0], g[2] if len(g) > 2 else 0)))
    gains = os.path.join(str(directory), "gains_%s.info" % tag); open(gains, "w").write("\n".join(lines + ["}", ""]))
    return task, gains


def distinct_rows(handle_row, n, seed=5):
    """n distinct rows around handle_row: row 0 is handle_row itself, the others scale every field by its own factor in [0.5, 1.5] and set the friction
    coefficients to one of 0.15 / 0.3 / 0.6 / 0.9"""
    rng = np.random.default_rng(seed); rows = np.repeat(np.asarray(handle_row, dtype=np.float64)[None], n, axis=0)
    for r in range(1, n):
        rows[r] *= rng.uniform(0.5, 1.5, rows.shape[1])
        rows[r, L["friction_mu"][0]] = (0.15, 0.3, 0.6, 0.9)[r % 4]; rows[r, L["wbc_friction"][0]] = (0.6, 0.15, 0.9, 0.3)[r % 4]
    return rows
