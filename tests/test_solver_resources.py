"""Compiled footprint of the XPBD solve kernels (CPU only: reads the sm_90a object).

The solves are latency bound per world: each substep lasts as long as the slowest
world's dependent chain in each wave of resident worlds, so the kernels are sized
so that room's 8192 worlds need as few waves as possible on an H100 (132 SMs).
This reads `cuobjdump -res-usage` of the `make` build and checks that no solve
uses a stack or local memory, and how many worlds its registers and shared memory
keep resident."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "madrona_b200", "build", "kernels_physics.o")

# H100 SXM (sm_90): per-SM limits
SMS = 132
REGS_PER_SM = 65536
REG_ALLOC_UNIT = 256          # registers per warp are allocated in units of 256
MAX_WARPS_PER_SM = 64
MAX_BLOCKS_PER_SM = 32
SHARED_PER_SM = 233472        # 228 KB, with the carveout at its maximum
SHARED_ALLOC_UNIT = 128
BLOCK_THREADS = 64            # kPhysWorldThreads
ROOM_WORLDS = 8192


def _res_usage():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(OBJ) or not os.path.exists(cuobjdump):
        pytest.skip("needs the make build of kernels_physics.o and cuobjdump")
    out = subprocess.run([cuobjdump, "-res-usage", OBJ], capture_output=True, text=True, check=True).stdout
    usage, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
            continue
        if fn and "REG:" in line:
            usage[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            fn = None
    return usage


def _kernels(usage, name):
    hits = {k: v for k, v in usage.items() if name in k}
    assert hits, (name, sorted(usage))
    return hits


def _blocks_per_sm(res):
    warps = BLOCK_THREADS // 32
    regs_per_warp = -(-res["REG"] * 32 // REG_ALLOC_UNIT) * REG_ALLOC_UNIT
    by_regs = REGS_PER_SM // (regs_per_warp * warps)
    # cuobjdump's SHARED includes the 1 KB the driver reserves per block
    by_shared = SHARED_PER_SM // (-(-res["SHARED"] // SHARED_ALLOC_UNIT) * SHARED_ALLOC_UNIT)
    return min(by_regs, by_shared, MAX_WARPS_PER_SM // warps, MAX_BLOCKS_PER_SM)


@pytest.mark.parametrize("kernel", ["physSolvePositionsKernel", "physSolveVelocitiesKernel"])
def test_solve_has_no_stack_or_local_memory(kernel):
    for name, res in _kernels(_res_usage(), kernel).items():
        assert res["STACK"] == 0 and res["LOCAL"] == 0, (name, res)


@pytest.mark.parametrize("lanes", [16, 8])
def test_velocity_solve_blocks_per_sm(lanes):
    # velocitySolveLanes counts on kVelSolveBlocksPerSM = 8 blocks of either instance
    # per SM; at 8 lanes that holds room's 8192 worlds in one wave
    res = _kernels(_res_usage(), "physSolveVelocitiesKernelILi%dE" % lanes)
    (res,) = res.values()
    assert _blocks_per_sm(res) >= 8, res
    if lanes == 8:
        assert SMS * _blocks_per_sm(res) * (BLOCK_THREADS // lanes) >= ROOM_WORLDS, res


def test_position_solve_keeps_eight_blocks_per_sm():
    # 16 lanes per world at 115 registers: 8 blocks of 4 worlds per SM, 4224 worlds
    # resident, so room's 8192 worlds take two waves of this kernel
    (res,) = _kernels(_res_usage(), "physSolvePositionsKernel").values()
    assert _blocks_per_sm(res) >= 8, res
