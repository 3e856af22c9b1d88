from __future__ import annotations

import os
import struct
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Sequence, Tuple

import numpy as np

_ROOT = os.path.dirname(os.path.abspath(__file__))


@dataclass
class Slot:
    slot: int
    name: str
    dtype: str                 # numpy dtype name
    per_world: Tuple[int, ...]  # shape of one world's rows (fixed tables) / of one row (dynamic)
    dynamic: bool = False      # rows = live rows of a dynamic table (varies per step)


@dataclass
class SimDesc:
    name: str
    sources: List[str]
    num_exports: int
    num_taskgraphs: int
    inputs: List[Slot]
    outputs: List[Slot]
    # (cfg dict) -> bytes of the simulator's Config struct
    pack_config: Callable[[Dict], bytes]
    # (world index, cfg dict) -> bytes of one WorldInit struct
    pack_init: Callable[[int, Dict], bytes]
    # extra args for the oracle harness (--x0 .. --x3)
    oracle_extra: Callable[[Dict], List[int]]
    defaults: Dict = field(default_factory=dict)
    # () -> (blob, relocs): ObjectManager blob whose address goes into Config
    objects: Callable = None
    # extra NVRTC flags (e.g. a build variant of the same sources)
    compile_flags: List[str] = field(default_factory=list)
    # batch ray-cast renderer: (cfg) -> (mb2_render_config, keep_alive) or None
    render: Callable = None
    # (cfg, gpu_id) -> madrona_b200.Navmesh shared by all worlds; its 40-byte view goes
    # into cfg["_navmesh_view"] for pack_config
    navmesh: Callable = None


def _cartpole_cfg(cfg):
    return struct.pack("<I", int(cfg.get("max_steps", 200)))


def _cartpole_init(w, cfg):
    return struct.pack("<I", int(cfg.get("seed", 0)) + w)


def _grid_cfg(cfg):
    return struct.pack("<iii", int(cfg["grid_size"]), int(cfg["episode_len"]), int(cfg["init_items"]))


def _grid_init(w, cfg):
    return struct.pack("<I", int(cfg.get("seed", 0)) + w)


def _customnodes_init(w, cfg):
    return struct.pack("<II", int(cfg.get("seed", 0)) + w, 1 if w % 7 == 3 else 0)


def _navmesh_shared(cfg, gpu_id):
    import madrona_b200 as mb
    from .navmesh_plan import SHARED_PLAN_SEED, make_plan
    verts, polys = make_plan(SHARED_PLAN_SEED)
    return mb.Navmesh(verts, polys, gpu_id)


def _navmesh_cfg(cfg):
    flags = (1 if cfg.get("per_world", True) else 0) | (2 if cfg.get("bad_polygon", False) else 0)
    return bytes(cfg["_navmesh_view"]) + struct.pack("<II", int(cfg["episode_len"]), flags)


def _room_cfg(cfg):
    return struct.pack("<QII", int(cfg.get("obj_mgr_ptr", 0)), int(cfg["episode_len"]),
                       int(cfg.get("grab_period", 0)))


def _room_init(w, cfg):
    return struct.pack("<I", int(cfg.get("seed", 0)) + w)


def _room_objects():
    from .objects import room_objects
    return room_objects()


def _balls_objects():
    from .objects import balls_objects
    return balls_objects()


def _arena_objects():
    from .objects import arena_objects
    return arena_objects()


def _triggers_objects():
    from .objects import triggers_objects
    return triggers_objects()


def _image_size(cfg, default_res):
    """Render config image size from the fixture config: keyword arguments for the
    render_assets builders.  `width` and `height` (both) give non-square images, else the
    `resolution` square."""
    if "width" in cfg or "height" in cfg:
        return {"resolution": 0, "width": int(cfg.get("width", 0)), "height": int(cfg.get("height", 0))}
    return {"resolution": int(cfg.get("resolution", default_res))}


def _room_render_cfg(cfg):
    from .render_assets import make_render_config
    return make_render_config(rgbd=bool(cfg.get("rgbd", False)), gpu_id=int(cfg.get("_gpu_id", 0)),
                              **_image_size(cfg, 64))


SIMS: Dict[str, SimDesc] = {
    # GPU-only: custom-key SortArchetypeNode, checked against oracle/restate.py
    "sortcheck": SimDesc(
        name="sortcheck",
        sources=[os.path.join(_ROOT, "sortcheck", "sim.cpp")],
        num_exports=4,
        num_taskgraphs=1,
        inputs=[],
        outputs=[Slot(0, "key", "uint32", (1,), dynamic=True),
                 Slot(1, "payload", "uint32", (4,), dynamic=True),
                 Slot(2, "tag", "uint8", (6,), dynamic=True)],
        pack_config=lambda cfg: struct.pack("<II", int(cfg["items_per_world"]), int(cfg["key_mask"])),
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [],
        defaults={"items_per_world": 9, "key_mask": 0xFFFFFFFF, "seed": 0},
    ),
    # GPU only: sort / compaction at tile, pass and column-width edges (tests/test_sort_sweep.py);
    # per-world lists init_counts / creates / kill_steps (kill step 0 = never)
    "sortsweep": SimDesc(
        name="sortsweep",
        sources=[os.path.join(_ROOT, "sortsweep", "sim.cpp")],
        num_exports=10,
        num_taskgraphs=1,
        inputs=[],
        outputs=[Slot(0, "entity", "int32", (2,), dynamic=True),
                 Slot(1, "uid", "uint32", (1,), dynamic=True),
                 Slot(2, "key4", "uint32", (1,), dynamic=True),
                 Slot(3, "check", "uint32", (1,), dynamic=True),
                 Slot(4, "p2", "uint8", (2,), dynamic=True),
                 Slot(5, "p3", "uint8", (3,), dynamic=True),
                 Slot(6, "p12", "uint8", (12,), dynamic=True),
                 Slot(7, "p24", "uint8", (24,), dynamic=True),
                 Slot(8, "p48", "uint8", (48,), dynamic=True),
                 Slot(9, "summary", "uint32", (2,))],
        pack_config=lambda cfg: struct.pack("<IIII", int(cfg["shape"]), int(cfg["key_mode"]),
                                            int(cfg["sort_on_key8"]), int(cfg["destroy_threshold"])),
        pack_init=lambda w, cfg: struct.pack("<IIII", int(cfg.get("seed", 0)) + w, int(cfg["init_counts"][w]),
                                             int(cfg["creates"][w]), int(cfg["kill_steps"][w])),
        oracle_extra=lambda cfg: [],
        defaults={"shape": 0, "key_mode": 0, "sort_on_key8": 0, "destroy_threshold": 0, "seed": 0,
                  "init_counts": [9], "creates": [0], "kill_steps": [0]},
    ),
    "room": SimDesc(
        name="room",
        sources=[os.path.join(_ROOT, "room", "sim.cpp")],
        num_exports=13,
        num_taskgraphs=1,
        inputs=[Slot(0, "reset", "int32", (1,)), Slot(1, "action", "int32", (2, 3))],
        outputs=[Slot(2, "reward", "float32", (2,)), Slot(3, "done", "int32", (2,)),
                 Slot(4, "self_obs", "float32", (2, 9)), Slot(5, "lidar", "float32", (2, 16, 2)),
                 Slot(6, "agent_pos", "float32", (2, 3)), Slot(7, "agent_rot", "float32", (2, 4)),
                 Slot(8, "body_count", "int32", (1,)),
                 Slot(9, "body_pos", "float32", (3,), dynamic=True),
                 Slot(10, "body_rot", "float32", (4,), dynamic=True),
                 Slot(11, "body_entity", "int32", (2,), dynamic=True),
                 Slot(12, "body_vel", "float32", (6,), dynamic=True)],
        pack_config=_room_cfg,
        pack_init=_room_init,
        oracle_extra=lambda cfg: [int(cfg["episode_len"]), int(cfg.get("seed", 0)),
                                  int(cfg.get("grab_period", 0))],
        defaults={"episode_len": 100, "seed": 0, "grab_period": 0},
        objects=_room_objects,
    ),
    # Hide&Seek-class arena (BASELINE configs[2]): 49 bodies, 6 agents, wedge / hexagonal hulls,
    # hinge joints (doors) + fixed joints (grab), entity churn on every episode reset
    "arena": SimDesc(
        name="arena",
        sources=[os.path.join(_ROOT, "arena", "sim.cpp")],
        num_exports=15,
        num_taskgraphs=1,
        inputs=[Slot(0, "reset", "int32", (1,)), Slot(1, "action", "int32", (6, 4))],
        outputs=[Slot(2, "reward", "float32", (6,)), Slot(3, "done", "int32", (6,)),
                 Slot(4, "self_obs", "float32", (6, 10)), Slot(5, "other_obs", "float32", (6, 5, 4)),
                 Slot(6, "lidar", "float32", (6, 16, 2)),
                 Slot(7, "agent_pos", "float32", (6, 3)), Slot(8, "agent_rot", "float32", (6, 4)),
                 Slot(9, "body_count", "int32", (1,)), Slot(10, "joint_count", "int32", (1,)),
                 Slot(11, "body_pos", "float32", (3,), dynamic=True),
                 Slot(12, "body_rot", "float32", (4,), dynamic=True),
                 Slot(13, "body_entity", "int32", (2,), dynamic=True),
                 Slot(14, "body_vel", "float32", (6,), dynamic=True)],
        pack_config=lambda cfg: struct.pack("<QII", int(cfg.get("obj_mgr_ptr", 0)),
                                            int(cfg["episode_len"]), 0),
        pack_init=_room_init,
        oracle_extra=lambda cfg: [int(cfg["episode_len"]), int(cfg.get("seed", 0))],
        defaults={"episode_len": 100, "seed": 0},
        objects=_arena_objects,
    ),
    # the room fixture with Solver::TGS (the reference's TGS is a collision-free integrator)
    "room_tgs": SimDesc(
        name="room_tgs",
        sources=[os.path.join(_ROOT, "room", "sim.cpp")],
        num_exports=13,
        num_taskgraphs=1,
        inputs=[Slot(0, "reset", "int32", (1,)), Slot(1, "action", "int32", (2, 3))],
        outputs=[Slot(2, "reward", "float32", (2,)), Slot(3, "done", "int32", (2,)),
                 Slot(4, "self_obs", "float32", (2, 9)), Slot(5, "lidar", "float32", (2, 16, 2)),
                 Slot(6, "agent_pos", "float32", (2, 3)), Slot(7, "agent_rot", "float32", (2, 4)),
                 Slot(8, "body_count", "int32", (1,)),
                 Slot(9, "body_pos", "float32", (3,), dynamic=True),
                 Slot(10, "body_rot", "float32", (4,), dynamic=True),
                 Slot(11, "body_entity", "int32", (2,), dynamic=True),
                 Slot(12, "body_vel", "float32", (6,), dynamic=True)],
        pack_config=_room_cfg,
        pack_init=_room_init,
        oracle_extra=lambda cfg: [int(cfg["episode_len"]), int(cfg.get("seed", 0)),
                                  int(cfg.get("grab_period", 0))],
        defaults={"episode_len": 100, "seed": 0, "grab_period": 0},
        objects=_room_objects,
        compile_flags=["-DROOM_TGS=1"],
    ),
    # the room fixture built with -DROOM_ENABLE_RENDER=1 (BASELINE configs[3]); GPU only:
    # the reference CPU backend cannot ray cast (src/render/ecs_system.cpp:684-689)
    "room_render": SimDesc(
        name="room_render",
        sources=[os.path.join(_ROOT, "room", "sim.cpp")],
        num_exports=17,
        num_taskgraphs=1,
        inputs=[Slot(0, "reset", "int32", (1,)), Slot(1, "action", "int32", (2, 3))],
        outputs=[Slot(2, "reward", "float32", (2,)), Slot(3, "done", "int32", (2,)),
                 Slot(6, "agent_pos", "float32", (2, 3)), Slot(7, "agent_rot", "float32", (2, 4)),
                 Slot(8, "body_count", "int32", (1,)),
                 Slot(9, "body_pos", "float32", (3,), dynamic=True),
                 Slot(10, "body_rot", "float32", (4,), dynamic=True)],
        pack_config=_room_cfg,
        pack_init=_room_init,
        oracle_extra=lambda cfg: [],
        defaults={"episode_len": 100, "seed": 0, "grab_period": 0, "resolution": 64, "rgbd": False},
        objects=_room_objects,
        compile_flags=["-DROOM_ENABLE_RENDER=1"],
        render=_room_render_cfg,
    ),
    # spheres: sphere-sphere / sphere-plane / sphere-hull (GJK) contacts, physics only
    "balls": SimDesc(
        name="balls",
        sources=[os.path.join(_ROOT, "balls", "sim.cpp")],
        num_exports=4,
        num_taskgraphs=1,
        inputs=[],
        outputs=[Slot(0, "body_pos", "float32", (16, 3)), Slot(1, "body_rot", "float32", (16, 4)),
                 Slot(2, "body_vel", "float32", (16, 6)), Slot(3, "body_entity", "int32", (16, 2))],
        pack_config=lambda cfg: struct.pack("<Q", int(cfg.get("obj_mgr_ptr", 0))),
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [int(cfg.get("seed", 0))],
        defaults={"seed": 0},
        objects=_balls_objects,
    ),
    # build variant with 95 bodies per world (more than one 64-bit word of leaf masks)
    "balls_many": SimDesc(
        name="balls_many",
        sources=[os.path.join(_ROOT, "balls", "sim.cpp")],
        num_exports=4,
        num_taskgraphs=1,
        inputs=[],
        outputs=[Slot(0, "body_pos", "float32", (95, 3)), Slot(1, "body_rot", "float32", (95, 4)),
                 Slot(2, "body_vel", "float32", (95, 6)), Slot(3, "body_entity", "int32", (95, 2))],
        pack_config=lambda cfg: struct.pack("<Q", int(cfg.get("obj_mgr_ptr", 0))),
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [int(cfg.get("seed", 0))],
        defaults={"seed": 0},
        objects=_balls_objects,
        compile_flags=["-DBALLS_MANY=1"],
    ),
    # GPU only: batch ray caster with a real TLAS / BLAS, materials, lights (tests/test_render_bvh.py)
    "gallery": SimDesc(
        name="gallery",
        sources=[os.path.join(_ROOT, "gallery", "sim.cpp")],
        num_exports=10,
        num_taskgraphs=1,
        inputs=[],
        outputs=[],
        pack_config=lambda cfg: struct.pack("<II", int(cfg["num_props"]), 5),
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [],
        defaults={"num_props": 100, "seed": 0, "resolution": 40, "rgbd": True},
        render=lambda cfg: __import__("sims.render_assets", fromlist=["x"]).make_gallery_render_config(
            rgbd=bool(cfg.get("rgbd", True)), gpu_id=int(cfg.get("_gpu_id", 0)), **_image_size(cfg, 40)),
    ),
    # GPU only: the gallery built with -DGALLERY_PER_WORLD=1: props[w] props in world w (every
    # 17th hidden, as in the gallery), layouts[w] 0 scattered / 1 clustered (deep Morton tree)
    "gallery_sized": SimDesc(
        name="gallery_sized",
        sources=[os.path.join(_ROOT, "gallery", "sim.cpp")],
        num_exports=10,
        num_taskgraphs=1,
        inputs=[],
        outputs=[],
        pack_config=lambda cfg: struct.pack("<II", 0, 5),
        pack_init=lambda w, cfg: struct.pack("<III", int(cfg.get("seed", 0)) + w, int(cfg["props"][w]),
                                             int(cfg["layouts"][w]) if cfg.get("layouts") else 0),
        oracle_extra=lambda cfg: [],
        defaults={"props": [100], "layouts": None, "seed": 0, "resolution": 40, "rgbd": True},
        compile_flags=["-DGALLERY_PER_WORLD=1"],
        render=lambda cfg: __import__("sims.render_assets", fromlist=["x"]).make_gallery_render_config(
            rgbd=bool(cfg.get("rgbd", True)), gpu_id=int(cfg.get("_gpu_id", 0)), **_image_size(cfg, 40)),
    ),
    # GPU only: the gallery sim with uvs and textured materials (tests/test_render_textures.py);
    # same sources and flags, so it shares the gallery's simulator module
    "gallery_textured": SimDesc(
        name="gallery_textured",
        sources=[os.path.join(_ROOT, "gallery", "sim.cpp")],
        num_exports=10,
        num_taskgraphs=1,
        inputs=[],
        outputs=[],
        pack_config=lambda cfg: struct.pack("<II", int(cfg["num_props"]), 5),
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [],
        defaults={"num_props": 100, "seed": 0, "resolution": 40, "rgbd": True, "bc7": False},
        render=lambda cfg: __import__("sims.render_assets", fromlist=["x"]).make_gallery_textured_render_config(
            rgbd=bool(cfg.get("rgbd", True)), gpu_id=int(cfg.get("_gpu_id", 0)),
            bc7=bool(cfg.get("bc7", False)), **_image_size(cfg, 40)),
    ),
    # GPU only: 145 bodies per world, past the per-world body cap (tests/test_cliffs.py)
    "balls_cliff": SimDesc(
        name="balls_cliff",
        sources=[os.path.join(_ROOT, "balls", "sim.cpp")],
        num_exports=4,
        num_taskgraphs=1,
        inputs=[],
        outputs=[Slot(0, "body_pos", "float32", (145, 3))],
        pack_config=lambda cfg: struct.pack("<Q", int(cfg.get("obj_mgr_ptr", 0))),
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [int(cfg.get("seed", 0))],
        defaults={"seed": 0},
        objects=_balls_objects,
        compile_flags=["-DBALLS_MANY=2"],
    ),
    # broadphase without the solver: standalone overlap rows (CandidateCollision), zone
    # queries (findEntitiesWithinAABB / checkEntityAABBOverlap), a two-hull compound, a
    # sphere, pickups destroyed and recreated (tests/test_overlap_queries.py)
    "triggers": SimDesc(
        name="triggers",
        sources=[os.path.join(_ROOT, "triggers", "sim.cpp")],
        num_exports=7,
        num_taskgraphs=1,
        inputs=[Slot(0, "action", "int32", (2, 2))],
        outputs=[Slot(1, "pairs", "int32", (1 + 32 * 4,)), Slot(2, "zone", "int32", (8,)),
                 Slot(3, "agent_pos", "float32", (2, 3)),
                 Slot(4, "pickup_entity", "int32", (2,), dynamic=True),
                 Slot(5, "pickup_pos", "float32", (3,), dynamic=True),
                 Slot(6, "prop_entity", "int32", (7, 2))],
        pack_config=lambda cfg: struct.pack("<Q", int(cfg.get("obj_mgr_ptr", 0))),
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [int(cfg.get("seed", 0))],
        defaults={"seed": 0},
        objects=_triggers_objects,
    ),
    # pressure plates after the XPBD step: findEntitiesWithinAABB on the refitted tree,
    # checkEntityAABBOverlap goal zone, doors (static bodies) that follow their buttons,
    # a sphere resting on a button, episode resets (tests/test_overlap_queries.py)
    "buttons": SimDesc(
        name="buttons",
        sources=[os.path.join(_ROOT, "buttons", "sim.cpp")],
        num_exports=8,
        num_taskgraphs=1,
        inputs=[Slot(0, "reset", "int32", (1,)), Slot(1, "action", "int32", (2, 3))],
        outputs=[Slot(2, "button_state", "int32", (2, 4)), Slot(3, "door_pos", "float32", (2, 3)),
                 Slot(4, "agent_pos", "float32", (2, 3)), Slot(5, "goal", "int32", (2,)),
                 Slot(6, "body_pos", "float32", (3,), dynamic=True),
                 Slot(7, "body_entity", "int32", (2,), dynamic=True)],
        pack_config=lambda cfg: struct.pack("<QII", int(cfg.get("obj_mgr_ptr", 0)),
                                            int(cfg["episode_len"]), 0),
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [int(cfg["episode_len"]), int(cfg.get("seed", 0))],
        defaults={"episode_len": 100, "seed": 0},
        objects=_balls_objects,
    ),
    # GPU only: the triggers graph plus setupPhysicsStepTasks, rejected at launch-graph build
    "triggers_with_solver": SimDesc(
        name="triggers_with_solver",
        sources=[os.path.join(_ROOT, "triggers", "sim.cpp")],
        num_exports=7,
        num_taskgraphs=1,
        inputs=[Slot(0, "action", "int32", (2, 2))],
        outputs=[Slot(2, "zone", "int32", (8,))],
        pack_config=lambda cfg: struct.pack("<Q", int(cfg.get("obj_mgr_ptr", 0))),
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [],
        defaults={"seed": 0},
        objects=_triggers_objects,
        compile_flags=["-DTRIGGERS_WITH_SOLVER=1"],
    ),
    "gridworld": SimDesc(
        name="gridworld",
        sources=[os.path.join(_ROOT, "gridworld", "sim.cpp")],
        num_exports=10,
        num_taskgraphs=1,
        inputs=[Slot(0, "reset", "int32", (1,)), Slot(1, "action", "int32", (2,))],
        outputs=[Slot(2, "agent_pos", "int32", (2, 2)), Slot(3, "reward", "float32", (2,)),
                 Slot(4, "obs", "int32", (2, 4)), Slot(5, "item_count", "int32", (1,)),
                 Slot(9, "done", "int32", (1,)),
                 Slot(6, "item_pos", "int32", (2,), dynamic=True),
                 Slot(7, "item_entity", "int32", (2,), dynamic=True),
                 Slot(8, "item_kind", "int32", (1,), dynamic=True)],
        pack_config=_grid_cfg,
        pack_init=_grid_init,
        oracle_extra=lambda cfg: [int(cfg["grid_size"]), int(cfg["episode_len"]),
                                  int(cfg["init_items"]), int(cfg.get("seed", 0))],
        defaults={"grid_size": 8, "episode_len": 50, "init_items": 6, "seed": 0},
    ),
    # custom task-graph nodes: addNodeFn (fixed counts, 1 / 32 / 256 threads per invocation),
    # addDynamicCountNode, addOneOffNode, node data, a second task graph (tests/test_custom_nodes.py);
    # world w never has tokens when w % 7 == 3
    "customnodes": SimDesc(
        name="customnodes",
        sources=[os.path.join(_ROOT, "customnodes", "sim.cpp")],
        num_exports=8,
        num_taskgraphs=2,
        inputs=[],
        outputs=[Slot(0, "world_sum", "uint32", (4,)), Slot(1, "coop", "uint32", (7,)),
                 Slot(2, "census", "uint32", (4,)),
                 Slot(3, "token_entity", "int32", (2,), dynamic=True),
                 Slot(4, "token_val", "uint32", (1,), dynamic=True),
                 Slot(5, "token_out", "uint32", (1,), dynamic=True)],
        pack_config=lambda cfg: struct.pack("<IIII", 0, 0, 0, 0),
        pack_init=_customnodes_init,
        oracle_extra=lambda cfg: [int(cfg.get("seed", 0))],
        defaults={"seed": 0},
    ),
    # GPU only: the same fixture with the ParallelForNode twin of its dynamic-count node
    # (scripts/bench_custom_nodes.py); it computes the same columns
    "customnodes_bench": SimDesc(
        name="customnodes_bench",
        sources=[os.path.join(_ROOT, "customnodes", "sim.cpp")],
        num_exports=8,
        num_taskgraphs=2,
        inputs=[],
        outputs=[Slot(0, "world_sum", "uint32", (4,)), Slot(1, "coop", "uint32", (7,)),
                 Slot(5, "token_out", "uint32", (1,), dynamic=True)],
        pack_config=lambda cfg: struct.pack("<IIII", 0, 0, 0, 0),
        pack_init=_customnodes_init,
        oracle_extra=lambda cfg: [],
        defaults={"seed": 0},
        compile_flags=["-DCUSTOMNODES_BENCH=1"],
    ),
    # GPU only: invocation probe -- a node with fixed count `count` (0: dynamic) and `threads`
    # threads per invocation records its runs in 4096 rows (invocation i -> row i % 4096);
    # dynamic=1 sets the count from a one-off node and has invocation 0 zero it while it runs
    "customnodes_probe": SimDesc(
        name="customnodes_probe",
        sources=[os.path.join(_ROOT, "customnodes", "sim.cpp")],
        num_exports=8,
        num_taskgraphs=2,
        inputs=[],
        outputs=[Slot(6, "probe", "uint32", (14,), dynamic=True), Slot(7, "probe_info", "uint32", (2,))],
        pack_config=lambda cfg: struct.pack("<IIII", int(cfg["count"]), int(cfg["threads"]),
                                            int(cfg["dynamic"]), int(cfg["extra_node_datas"])),
        pack_init=_customnodes_init,
        oracle_extra=lambda cfg: [],
        defaults={"count": 1, "threads": 1, "dynamic": 0, "extra_node_datas": 0, "seed": 0},
        compile_flags=["-DCUSTOMNODES_PROBE=1"],
    ),
    # navigation meshes: a navmesh per world built in the world constructor and one shared
    # through Config; agents walk Dijkstra fields towards sampled goals and count what a
    # predicated BFS reaches (tests/test_navmesh.py).  per_world=False: every agent walks the
    # shared mesh; bad_polygon=True: world 1's plan has a 2-vertex polygon
    "navmesh": SimDesc(
        name="navmesh",
        sources=[os.path.join(_ROOT, "navmesh", "sim.cpp")],
        num_exports=7,
        num_taskgraphs=1,
        inputs=[],
        outputs=[Slot(0, "pos", "float32", (6, 3)), Slot(1, "poly", "uint32", (6,)),
                 Slot(2, "dist", "float32", (6,)), Slot(3, "dijkstra", "uint32", (6, 2)),
                 Slot(4, "bfs", "uint32", (6, 2)), Slot(5, "goal", "uint32", (6, 4)),
                 Slot(6, "mesh", "uint32", (6,))],
        pack_config=_navmesh_cfg,
        pack_init=lambda w, cfg: struct.pack("<I", int(cfg.get("seed", 0)) + w),
        oracle_extra=lambda cfg: [int(cfg["episode_len"]), int(cfg.get("seed", 0)),
                                  1 if cfg.get("per_world", True) else 0],
        defaults={"episode_len": 40, "seed": 0, "per_world": True, "bad_polygon": False},
        navmesh=_navmesh_shared,
    ),
    "cartpole": SimDesc(
        name="cartpole",
        sources=[os.path.join(_ROOT, "cartpole", "sim.cpp")],
        num_exports=5,
        num_taskgraphs=1,
        inputs=[Slot(0, "reset", "int32", (1,)), Slot(1, "action", "int32", (1,))],
        outputs=[Slot(2, "state", "float32", (4,)), Slot(3, "reward", "float32", (1,)),
                 Slot(4, "done", "int32", (1,))],
        pack_config=_cartpole_cfg,
        pack_init=_cartpole_init,
        oracle_extra=lambda cfg: [int(cfg.get("max_steps", 200)), int(cfg.get("seed", 0))],
        defaults={"max_steps": 200, "seed": 0},
    ),
}


def pack_world_inits(desc: SimDesc, num_worlds: int, cfg: Dict) -> bytes:
    return b"".join(desc.pack_init(w, cfg) for w in range(num_worlds))


def make_executor(name: str, num_worlds: int, gpu_id: int = 0, objects_fn=None, **cfg):
    """Build a madrona_b200.MWCudaExecutor for a fixture sim (needs an H100).
    objects_fn overrides the fixture's ObjectManager (same object indices): it returns either
    a (blob, relocations) pair or a madrona_b200.RigidBodyAssets built on this GPU."""
    import madrona_b200 as mb

    desc = SIMS[name]
    full = dict(desc.defaults)
    full.update(cfg)
    keep_alive = None
    made = None
    if desc.objects is not None:
        made = (objects_fn or desc.objects)()
        if isinstance(made, mb.RigidBodyAssets):
            full["obj_mgr_ptr"] = made.device_ptr
            keep_alive = made
            made = None
    if made is not None:
        # upload the ObjectManager blob and relocate its pointers to device addresses
        import numpy as np
        import torch
        from .objects import relocate
        blob, relocs = made
        dev_buf = torch.empty(len(blob) + 64, dtype=torch.uint8, device=f"cuda:{gpu_id}")
        base = (dev_buf.data_ptr() + 63) // 64 * 64
        fixed = relocate(blob, relocs, base)
        start = base - dev_buf.data_ptr()
        dev_buf[start:start + len(fixed)].copy_(torch.from_numpy(np.frombuffer(fixed, dtype=np.uint8).copy()))
        torch.cuda.synchronize(gpu_id)
        full["obj_mgr_ptr"] = base
        keep_alive = dev_buf
    navmesh = None
    if desc.navmesh is not None:
        navmesh = desc.navmesh(full, gpu_id)
        full["_navmesh_view"] = navmesh.view_bytes()
    inits = pack_world_inits(desc, num_worlds, full)
    state = mb.StateConfig(
        worldInit=inits,
        numWorldInitBytes=len(inits) // num_worlds,
        userConfig=desc.pack_config(full),
        numWorldDataBytes=0,          # 0 => sizeof(Sim) as the device compiler sees it
        worldDataAlignment=16,
        numWorlds=num_worlds,
        numTaskGraphs=desc.num_taskgraphs,
        numExportedBuffers=desc.num_exports,
    )
    compile_cfg = mb.CompileConfig(userSources=desc.sources,
                                   userCompileFlags=["-I" + os.path.dirname(desc.sources[0])] +
                                   list(desc.compile_flags))
    full["_gpu_id"] = gpu_id
    render_cfg, render_keep = (desc.render(full) if desc.render is not None else (None, None))
    ex = mb.MWCudaExecutor(state, compile_cfg, gpu_id=gpu_id, render_cfg=render_cfg)
    ex._keep_alive = (keep_alive, render_keep, navmesh)
    return ex
