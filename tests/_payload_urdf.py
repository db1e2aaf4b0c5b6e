"""The model that a model payload stands for (qmb200_set_model_payload): the robot's URDF with an extra link fixed to the end-effector frame's link at
o_ee that carries m_ee, and one fixed to the base link at o_base that carries m_base, both point masses without rotational inertia.  Written to a
directory the caller owns (a pytest tmp_path); the files under assets/ and tests/fixtures/ are read, never written."""
import os
import re

from qm_control_b200 import _lib

EE_FRAME = "j2n6s300_end_effector"   # model_settings.eeFrame of qm_task.info
BASE_LINK = "base"


def _link(name, parent, mass, xyz):
    return ('  <link name="{n}">\n    <inertial>\n      <origin xyz="0 0 0" rpy="0 0 0"/>\n      <mass value="{m!r}"/>\n'
            '      <inertia ixx="0" ixy="0" ixz="0" iyy="0" iyz="0" izz="0"/>\n    </inertial>\n  </link>\n'
            '  <joint name="{n}_joint" type="fixed">\n    <parent link="{p}"/>\n    <child link="{n}"/>\n'
            '    <origin xyz="{x!r} {y!r} {z!r}" rpy="0 0 0"/>\n  </joint>\n').format(n=name, p=parent, m=float(mass), x=float(xyz[0]), y=float(xyz[1]), z=float(xyz[2]))


def edited_urdf(directory, payload, name="robot_payload.urdf"):
    """payload: 8 values in _lib.PAYLOAD_LAYOUT.  A zero mass adds no link.  → path of the edited URDF."""
    p = [float(v) for v in payload]; assert len(p) == 8
    src = open(_lib.asset("qm_robot.urdf")).read()
    assert re.search(r'<link name="%s"' % EE_FRAME, src) and re.search(r'<link name="%s"' % BASE_LINK, src)
    extra = ""
    if p[0] != 0.0:
        extra += _link("payload_ee", EE_FRAME, p[0], p[1:4])
    if p[4] != 0.0:
        extra += _link("payload_base", BASE_LINK, p[4], p[5:8])
    i = src.rindex("</robot>")
    path = os.path.join(str(directory), name)
    with open(path, "w") as f:
        f.write(src[:i] + extra + src[i:])
    return path
