"""The rollout export of the reference in the structure its tools consume (SURVEY 8f.2).

The reference renders a solve with `brax.io.html.render(sys, rollout)` (upstream mbd/utils.py:23-34,
mbd_planner.py:171-178) and `scripts/vis_diffusion.py:27-143` re-implements `brax.io.json.dumps` on the same inputs: a
`System` with MuJoCo-style geom arrays (`ngeom, geom_bodyid, geom_type, geom_pos, geom_quat, geom_size, geom_rgba`,
`link_names`) and a list of pipeline states with `.x.pos [L,3]` / `.x.rot [L,4]`.  Both end in ONE JSON document for the Brax
visualizer: `geoms` keyed by link name (plus "world"), `states.x.{pos,rot}` stacked over time, `opt.timestep` = the env dt,
`link_names`.  This module writes exactly that document from this package's own `System` / `PipelineState`s — no Brax needed
to produce it — plus the two-line HTML page Brax's `html.render` wraps around it (the viewer script is fetched from the
Brax repository's CDN by the browser, as in Brax's own page), and a thin adapter (`BraxLikeSystem`) exposing the geom arrays
so that `vis_diffusion.py`'s own `dumps` can walk them.
"""
from __future__ import annotations

import json
from typing import List, Sequence

import numpy as np

# brax.io.json._GEOM_TYPE_NAMES (mujoco mjtGeom numbering)
GEOM_TYPE_ID = {"plane": 0, "hfield": 1, "sphere": 2, "capsule": 3, "ellipsoid": 4, "cylinder": 5, "box": 6, "mesh": 7}
GEOM_TYPE_NAMES = {0: "Plane", 1: "HeightMap", 2: "Sphere", 3: "Capsule", 4: "Ellipsoid", 5: "Cylinder", 6: "Box", 7: "Mesh"}
VIEWER_JS = "https://cdn.jsdelivr.net/gh/google/brax@v0.10.5/brax/visualizer/js/viewer.js"


class BraxLikeSystem:
    """The attributes of a Brax `System` that `brax.io.json.dumps` / `vis_diffusion.py:dumps` read, built from `mjcf.System`."""

    def __init__(self, sys, dt: float):
        self.link_names = list(sys.link_names)
        self.dt = float(dt)
        geoms = list(sys.geoms)
        self.ngeom = len(geoms)
        self.geom_bodyid = np.array([g.body + 1 for g in geoms], dtype=np.int32)     # mujoco body ids: 0 = world
        self.geom_type = np.array([GEOM_TYPE_ID[g.type] for g in geoms], dtype=np.int32)
        self.geom_pos = np.array([g.pos for g in geoms], dtype=np.float32).reshape(-1, 3)
        self.geom_quat = np.array([g.quat for g in geoms], dtype=np.float32).reshape(-1, 4)
        size = np.zeros((self.ngeom, 3), np.float32)
        for i, g in enumerate(geoms):
            s = np.asarray(g.size, np.float32).ravel()[:3]
            size[i, :len(s)] = s
        self.geom_size = size
        self.geom_rgba = np.tile(np.float32([0.8, 0.6, 0.4, 1.0]), (self.ngeom, 1))
        self.geom_rgba[self.geom_type == 0] = np.float32([0.5, 0.5, 0.5, 1.0])
        for i, g in enumerate(geoms):           # models that carry their own colours (pushT: green pusher, blue T, red ghost)
            if getattr(g, "rgba", None) is not None:
                self.geom_rgba[i] = np.asarray(g.rgba, np.float32)


def _tolist(a):
    return np.asarray(a, dtype=np.float64).round(6).tolist()


def _link_geoms(bs: BraxLikeSystem):
    """-> (link names + "world", {link name: [geom dict]}): the geoms of the document, keyed by the name of their link"""
    link_names = [n or f"link {i}" for i, n in enumerate(bs.link_names)] + ["world"]
    link_geoms = {}
    for i in range(bs.ngeom):
        link_idx = int(bs.geom_bodyid[i]) - 1
        geom = {"name": GEOM_TYPE_NAMES[int(bs.geom_type[i])], "link_idx": link_idx, "pos": _tolist(bs.geom_pos[i]),
                "rot": _tolist(bs.geom_quat[i]), "rgba": _tolist(bs.geom_rgba[i]), "size": _tolist(bs.geom_size[i])}
        link_geoms.setdefault(link_names[link_idx], []).append(geom)
    return link_names, link_geoms


def to_dict(sys, pipeline_states: Sequence, dt: float) -> dict:
    """the document of `brax.io.json.dumps(sys.tree_replace({"opt.timestep": env.dt}), rollout)`"""
    bs = BraxLikeSystem(sys, dt)
    link_names, link_geoms = _link_geoms(bs)
    pos = np.stack([np.asarray(ps.x.pos, np.float32) for ps in pipeline_states])
    rot = np.stack([np.asarray(ps.x.rot, np.float32) for ps in pipeline_states])
    return {"link_names": link_names[:-1], "opt": {"timestep": float(dt)}, "dt": float(dt), "geoms": link_geoms,
            "states": {"x": {"pos": _tolist(pos), "rot": _tolist(rot)}}}


def dumps(sys, pipeline_states: Sequence, dt: float) -> str:
    return json.dumps(to_dict(sys, pipeline_states, dt))


def diffusion_to_dict(sys, pos, rot, dt: float, lift: bool = False) -> dict:
    """the document of `dumps` in the reference's scripts/vis_diffusion.py:27-112, from the world poses pos [K,T,L,3], rot [K,T,L,4]
    of K rollouts of T steps (one per diffusion iterate, the state before each step).

    Every link is drawn T times, copy k named `{name}_{k}` (k = 0 keeps the plain name) with its link_idx offset by k * L, so that
    one frame shows all T poses of a rollout.  Colours: world geoms as they are; `goal` links green (not offset: every copy sits on
    copy 0's pose); `_ref` links (humanoidtrack's reference bodies) torso / thigh fading green, the rest invisible; every other link
    fading red, from pale at k = 0 to full at k = T - 1.  Frames: one per rollout, then T frames that play the last rollout with
    every copy on that step's pose.  lift (pushT): step i is raised by i * 0.01 / 50 so that the copies do not overlap."""
    bs = BraxLikeSystem(sys, dt)
    link_names, link_geoms = _link_geoms(bs)
    pos, rot = np.asarray(pos, np.float32), np.asarray(rot, np.float32)
    K, T, L = pos.shape[:3]
    nl = len(link_names) - 1
    all_link_geoms, all_link_names = {}, []
    for k in range(T):
        a = k / T * 0.8 + 0.2
        for name, geoms in link_geoms.items():
            name = f"{name}_{k}" if k > 0 else name
            geoms_new = []
            for geom in geoms:
                g = dict(geom)
                if "world" in name:
                    g["link_idx"] = -1
                elif "goal" in name:
                    g["rgba"] = [0.0, 1.0, 0.0, 1.0]
                elif "_ref" in name:
                    if "torso" in name or "thigh" in name:
                        g["link_idx"] = geom["link_idx"] + k * nl
                        g["rgba"] = [1 - a, 1.0, 1 - a, 1.0]
                    else:
                        g["rgba"] = [1.0, 1.0, 1.0, 0.0]
                else:
                    g["link_idx"] = geom["link_idx"] + k * nl
                    g["rgba"] = [1.0, 1 - a, 1 - a, 1.0]
                geoms_new.append(g)
            all_link_geoms[name] = geoms_new
            all_link_names.append(name)
    if lift:
        z = np.float32([i * 0.01 / 50 for i in range(T)])
        pos = pos + np.stack([np.zeros_like(z), np.zeros_like(z), z], axis=-1)[None, :, None, :]
    fpos = np.concatenate([pos.reshape(K, T * L, 3), np.tile(pos[-1][:, None], (1, T, 1, 1)).reshape(T, T * L, 3)])
    frot = np.concatenate([rot.reshape(K, T * L, 4), np.tile(rot[-1][:, None], (1, T, 1, 1)).reshape(T, T * L, 4)])
    return {"link_names": all_link_names, "opt": {"timestep": float(dt)}, "dt": float(dt), "geoms": all_link_geoms,
            "states": {"x": {"pos": _tolist(fpos), "rot": _tolist(frot)}}}


def page(doc: str, height: int = 480) -> str:
    """the page `brax.io.html.render_from_json` returns: the JSON document embedded next to the Brax viewer module"""
    return ("<html><head><title>brax visualizer</title><style>body{margin:0;padding:0;}#brax-viewer{margin:0;padding:0;height:"
            f"{int(height)}px;}}</style></head><body><script type=\"application/javascript\">var system = {doc};</script>"
            "<div id=\"brax-viewer\"></div><script type=\"module\">"
            f"import {{Viewer}} from '{VIEWER_JS}';"
            "const domElement = document.getElementById('brax-viewer');var viewer = new Viewer(domElement, system);"
            "</script></body></html>")


def render(sys, pipeline_states: Sequence, dt: float, height: int = 480) -> str:
    """the page `brax.io.html.render` returns: the JSON document embedded next to the Brax viewer module"""
    return page(dumps(sys, pipeline_states, dt), height)
