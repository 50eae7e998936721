"""CPU test: the register-accumulator engine's kernels keep every value in registers.  Its epilogues stage a group of
shared-memory operands in registers ahead of the arithmetic; a spill to local memory would put a memory round trip
back into the chains the staging hides, so `cuobjdump -res-usage` of the built library must show no stack frame and no
local memory for the update_e / update_v kernels (the exact-swish fused init_e + part A table form, whose libdevice
expf / division need more registers, may keep at most 8 bytes)."""
import re
import subprocess

from dig_b200 import _lib


def _usage():
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found = {}
    for name, res in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out):
        m = re.search(r"sphere_update_e_h16_kernelILb(\d)ELi(\d)ELb(\d)E", name) or re.search(r"sphere_update_v_h16_kernelILb(\d)E", name)
        if m:
            kind = "e" if "update_e" in name else "v"
            found[(kind,) + tuple(int(x) for x in m.groups())] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", res)}
    return found


def test_register_engine_kernels_do_not_spill():
    usage = _usage()
    assert len([k for k in usage if k[0] == "e"]) == 14 and len([k for k in usage if k[0] == "v"]) == 2, sorted(usage)
    for key, res in usage.items():
        fast = key[1] == 1
        limit = 8 if key == ("e", 0, 4, 1) else 0      # exact swish, init_e + part A, table form
        assert res["LOCAL"] == 0, (key, res)
        assert res["STACK"] <= (0 if fast else limit), (key, res)
