"""The chain executor's stage-mask rules and its frame planning across every feature at once.

The rule matrix: every feature state (off, the grid, the selection, the motion-vector view, the debug view modes, WHITE_BASE_COLOR, the
environment map, the bounding box) with TAA on and off, against the full stage mask and a mask missing each stage in turn, in both
orders - the feature on and then the mask configured, the mask configured and then the feature's setter. Both orders give the same
answer; a refused call leaves the configuration and the next frame's LDR output as they were.

Every feature together: one schedule of overlapping stretches (the environment map as a cube and then a sphere, the bounding box, the
grid, the selection with a change of its id, the debug views, the motion-vector view with a new elapsed time every frame and a TAA-off
stretch) gives the same bytes and launch counts replayed from graphs as issued eagerly, and a second pass over it builds no graph."""
import ctypes as C
import itertools

import pytest
import torch

from diligentfx_b200 import capi, synth
from diligentfx_b200.chain import STAGE_ALL, STAGE_COMPOSE, STAGE_TAA, STAGE_TONEMAP, ChainConfig, PostProcessChain

pytestmark = pytest.mark.gpu

SD, EM, MI, SHADED = capi.VIEW_MODE_SCENE_DEPTH, capi.VIEW_MODE_EDGE_MAP, capi.VIEW_MODE_MESH_ID, capi.VIEW_MODE_SHADED
MV, WHITE = capi.VIEW_MODE_MOTION_VECTORS, capi.VIEW_MODE_WHITE_BASE_COLOR
OTHER = 3  # a renderer debug view that HnPostProcess.psh does not draw itself
GRID = capi.GRID_FLAG_PLANES | capi.GRID_FLAG_AXES
SPHERE = 3
VIEWS = {"scene depth": SD, "edge map": EM, "mesh id": MI, "other debug view": OTHER, "white base colour": WHITE}
DEBUG_VIEWS = [v for v in VIEWS if VIEWS[v] != WHITE]
FEATURES = ["off", "grid", "selection", "motion vectors", *VIEWS, "env map", "bound box"]
MASKS = [STAGE_ALL] + [STAGE_ALL & ~(1 << i) for i in range(7)]


# ---- the rule matrix ------------------------------------------------------------------------------------------------------------------
W, H = 64, 36


def _required(feature: str, disable_taa: int) -> int:
    """The stages the chain requires of its mask with `feature` on."""
    need = STAGE_COMPOSE | STAGE_TONEMAP if disable_taa else 0  # the TAA-off frame is drawn by the final compose
    if feature == "grid":
        need |= STAGE_TONEMAP
    elif feature == "motion vectors":
        need |= STAGE_COMPOSE | STAGE_TONEMAP
    elif not disable_taa and (feature == "selection" or feature in DEBUG_VIEWS):
        need |= STAGE_COMPOSE | STAGE_TAA
    return need


class _Features:
    """Switches one feature on through the C-ABI and returns the status."""

    def __init__(self):
        self.sel = torch.from_numpy(synth.selection_depth(W, H, 0, [SPHERE])).cuda()
        self.mesh = torch.from_numpy(synth.mesh_id(W, H, 0)).cuda()
        self.cube = [torch.from_numpy(l).cuda() for l in synth.env_map_cube(16, 3)]
        self.box = capi.BoundBoxAttribs.make(synth.sphere_bound_box(SPHERE), (1.0, 0.8, 0.2, 1.0))

    def set(self, ch: PostProcessChain, feature: str) -> int:
        L, c = ch.lib, ch.chain
        if feature == "off":
            return capi.DFX_OK
        if feature == "grid":
            return L.dfx_chain_set_coordinate_grid(c, C.c_uint32(GRID), None)
        if feature == "selection":
            return L.dfx_chain_set_selection(c, C.byref(capi.SelectionAttribs.default()), C.byref(capi.plane_of(self.sel)))
        if feature == "motion vectors":
            return L.dfx_chain_set_motion_vector_view(c, 1, C.c_float(1 / 60))
        if feature == "env map":
            return L.dfx_chain_set_environment_map(c, capi.ENV_MAP_TYPE_CUBE, C.byref(capi.pyramid_of(self.cube)), C.c_uint32(0), None)
        if feature == "bound box":
            return L.dfx_chain_set_bound_box(c, C.byref(self.box))
        mode = VIEWS[feature]
        mesh = C.byref(capi.plane_of(self.mesh)) if mode == MI else None
        return L.dfx_chain_set_view_mode(c, mode, mesh, C.c_float(0.0))


def _chain(mask: int, disable_taa: int) -> PostProcessChain:
    return PostProcessChain(W, H, ChainConfig(stages=mask, enable_taa=not disable_taa))


def _config(ch: PostProcessChain) -> bytes:
    cfg = capi.ChainConfigC()
    capi.check(ch.lib.dfx_chain_get_config(ch.chain, C.byref(cfg)))
    return bytes(cfg)


def _frame(ch: PostProcessChain, fr: dict):
    """The frame's LDR bytes over a sentinel (a mask without TONEMAP writes none), or the refusal of a mask the frame cannot run."""
    ch.ldr.fill_(-7.0)
    try:
        return ch.run_frame(fr).cpu().numpy().tobytes()
    except capi.DfxError as e:
        return str(e)


def test_stage_rules_in_both_orders(built):
    lib = capi.load()
    fx = _Features()
    seq = synth.generate_sequence(W, H, 2)
    refs = {}

    def reference(feature, mask, disable_taa):
        """Two frames of a chain that never saw the refused call."""
        k = (feature, mask, disable_taa)
        if k not in refs:
            ch = _chain(mask, disable_taa)
            assert fx.set(ch, feature) == capi.DFX_OK, k
            refs[k] = [_frame(ch, fr) for fr in seq]
            ch.close()
        return refs[k]

    for feature, disable_taa, mask in itertools.product(FEATURES, (0, 1), MASKS):
        tag = (feature, disable_taa, hex(mask))
        ok = not (_required(feature, disable_taa) & ~mask)
        want = capi.DFX_OK if ok else capi.DFX_ERR_INVALID_ARG

        # 1. the feature on, then the mask
        ch = _chain(STAGE_ALL, disable_taa)
        assert fx.set(ch, feature) == capi.DFX_OK, tag
        before = _config(ch)
        first = None if ok else _frame(ch, seq[0])
        cfg = capi.ChainConfigC.from_buffer_copy(before)
        cfg.stages = mask
        assert lib.dfx_chain_set_config(ch.chain, C.byref(cfg)) == want, tag
        if ok:
            assert _config(ch) == bytes(cfg), tag
        else:
            assert _config(ch) == before, tag
            assert [first, _frame(ch, seq[1])] == reference(feature, STAGE_ALL, disable_taa), tag
        ch.close()

        # 2. the mask, then the feature
        if disable_taa and (~mask & (STAGE_COMPOSE | STAGE_TONEMAP)):
            cfg = capi.ChainConfigC()
            lib.dfx_chain_config_default(C.byref(cfg))
            cfg.stages, cfg.disable_taa = mask, 1
            out = C.c_void_p()
            assert lib.dfx_chain_create(W, H, C.byref(cfg), C.byref(out)) == capi.DFX_ERR_INVALID_ARG, tag
            continue
        ch = _chain(mask, disable_taa)
        before = _config(ch)
        first = None if ok else _frame(ch, seq[0])
        assert fx.set(ch, feature) == want, tag
        if not ok:
            assert _config(ch) == before, tag
            assert [first, _frame(ch, seq[1])] == reference("off", mask, disable_taa), tag
        ch.close()


# ---- every feature together -----------------------------------------------------------------------------------------------------------
WA, HA, N = 96, 54, 30


def _schedule() -> list[dict]:
    """Frame k's features. Overlapping stretches, 14 distinct graph keys: below the 16 at which dfx_chain_set_config (the TAA-off
    stretch) drops the graph cache."""
    s = [dict(env=None, box=False, grid=False, sel=None, view=SHADED, taa=True) for _ in range(N)]

    def on(name, value, frames):
        for k in frames:
            s[k][name] = value

    on("grid", True, [*range(3, 10), *range(22, 26)])
    on("env", capi.ENV_MAP_TYPE_CUBE, range(3, 13))
    on("env", capi.ENV_MAP_TYPE_SPHERE, range(18, 26))
    on("box", True, range(10, 22))
    on("sel", 7, range(10, 13))
    on("sel", 9, range(13, 18))
    on("view", SD, range(14, 16))
    on("view", EM, [16])
    on("view", MI, [17])
    on("view", MV, range(18, 22))
    on("taa", False, range(22, 26))
    return s


class _Everything:
    def __init__(self):
        self.cube = [torch.from_numpy(l).cuda() for l in synth.env_map_cube(16, 3)]
        self.sphere = [torch.from_numpy(l).cuda() for l in synth.env_map_sphere(32, 16, 3)]
        self.box = synth.sphere_bound_box(SPHERE)
        self.sel_depth = [synth.selection_depth(WA, HA, k, [SPHERE]) for k in range(N)]
        self.ids = [synth.mesh_id(WA, HA, k) for k in range(N)]

    def run(self, ch: PostProcessChain, seq: list[dict], first: int):
        """Runs the schedule from frame index `first`: the LDR planes, the launches and whether each frame was replayed."""
        lib = capi.load()
        sel_t = torch.empty((HA, WA), dtype=torch.float32, device="cuda")
        ids_t = torch.empty((HA, WA), dtype=torch.float32, device="cuda")
        out, launches, replayed = [], [], []
        for k, (fr, x) in enumerate(zip(seq, _schedule())):
            if x["env"] is None:
                ch.set_environment_map(None)
            else:
                ch.set_environment_map(x["env"], self.cube if x["env"] == capi.ENV_MAP_TYPE_CUBE else self.sphere)
            ch.set_bound_box(self.box if x["box"] else None)
            ch.set_coordinate_grid(GRID if x["grid"] else 0)
            if x["sel"] is None:
                ch.set_selection(None)
            else:
                sel_t.copy_(torch.from_numpy(self.sel_depth[k]))
                a = capi.SelectionAttribs.default()
                a.selection_id = x["sel"]
                ch.set_selection(a, sel_t)
            if x["view"] == MV:
                ch.set_motion_vector_view(1 / (30 + k))
            else:
                ids_t.copy_(torch.from_numpy(self.ids[k]))
                ch.set_view_mode(x["view"], ids_t if x["view"] == MI else None)
            ch.cfg.enable_taa = x["taa"]
            n0, r0 = lib.dfx_launch_count(), ch.stats()["frames_replayed"]
            out.append(ch.run_frame(dict(fr, frame=first + k)).cpu().numpy().tobytes())
            launches.append(lib.dfx_launch_count() - n0)
            replayed.append(ch.stats()["frames_replayed"] > r0)
        return out, launches, replayed


def test_every_feature_together_replays_what_it_issues(built):
    seq = synth.generate_sequence(WA, HA, N)
    run = _Everything()
    eager = PostProcessChain(WA, HA, ChainConfig(graph=False))
    want, want_launches, _ = run.run(eager, seq, 0)
    assert eager.stats()["frames_replayed"] == 0
    eager.close()

    ch = PostProcessChain(WA, HA, ChainConfig(graph=True))
    got, launches, replayed = run.run(ch, seq, 0)
    for k in range(N):
        assert got[k] == want[k], (k, _schedule()[k])
    assert launches == want_launches
    stats = ch.stats()
    assert stats["graph_failures"] == 0 and 0 < stats["graphs_built"] < 16, stats
    assert sum(replayed) >= N // 2, replayed

    # the same schedule again, frame indices continuing: every key is cached, and only the first frame follows a different one
    _, _, again = run.run(ch, seq, N)
    assert ch.stats()["graphs_built"] == stats["graphs_built"], (stats, ch.stats())
    assert again[1:] == replayed[1:], (replayed, again)
    ch.close()
