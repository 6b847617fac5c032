"""Bone attachments held by the hierarchy (Hierarchy.setAttachments / propagateAttached / attachmentRounds, lb200_hierarchy_*attach*).

Every frame is held bit for bit to `AttachedWorld` below, a restatement of the frame World::setTransform (world.cpp:255-282, 337-342) and
RenderModuleImpl::onModelInstanceMoved / updateBoneAttachment (render_module.cpp:377-405, 1544-1566) make under the library's order: the
edits' closure is recomposed top-down (transformEntity's recursion through first_child / next_sibling), then the attachments run round by
round, each active one through oracle.bone_attachments and oracle.transform_compute_local, its subtree through oracle.transform_compose.
Globals of every node, locals of every node and the moved list are compared after every frame.
"""
import ctypes as C
import os

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes, sortkeys
from lumixengine_b200._lib import ERR_INVALID, ERR_STATE, LumixB200Error

pytestmark = pytest.mark.gpu
FIELDS = ("pos", "rot", "scale")


def _b(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(len(a), 56)


def _t(b):
    return np.ascontiguousarray(b).view(lb.TRANSFORM_DTYPE).reshape(-1)


def _bits_equal(a, b, what):
    for f in FIELDS:
        assert np.ascontiguousarray(a[f]).tobytes() == np.ascontiguousarray(b[f]).tobytes(), f"{what}: {f} differs"


def _random_transforms(rng, k, extent):
    t = np.zeros(k, lb.TRANSFORM_DTYPE)
    t["pos"] = (rng.random((k, 3)) * 2.0 - 1.0) * extent
    t["rot"] = scenes.random_unit_quats(rng, k)
    t["scale"] = (0.7 + 0.6 * rng.random((k, 3))).astype(np.float32)
    return t


def table_rounds(parents, attached, parent):
    """The library's order: X after Y when Y's attached node is an ancestor-or-self of X's parent node or a strict ancestor of X's attached
    node.  -> rounds (1-based), or None for a cycle."""
    att_of = {int(a): k for k, a in enumerate(attached)}
    m = len(attached)

    def above(q):
        out = []
        while q >= 0:
            if q in att_of:
                out.append(att_of[q])
            q = int(parents[q])
        return out

    deps = [above(int(parent[k])) + above(int(parents[attached[k]])) for k in range(m)]
    rounds = np.ones(m, np.int64)
    for _ in range(m + 2):
        new = np.array([1 + max([rounds[y] for y in deps[k]], default=0) for k in range(m)], np.int64)
        if (new > m).any():
            return None
        if np.array_equal(new, rounds):
            return rounds
        rounds = new
    return None


class AttachedWorld:
    """The oracle's hierarchy: globals G and locals L per node, the entity map and the attachment table."""

    def __init__(self, oracle, parents, locals_, roots, entity):
        self.o = oracle
        self.parents = np.asarray(parents, np.int64)
        self.n = len(parents)
        self.L = locals_.copy()
        self.G = _t(oracle.propagate(parents, _b(locals_), _b(roots)))
        self.entity = np.asarray(entity, np.int64)
        self.children = [[] for _ in range(self.n)]
        for i in range(self.n):
            if self.parents[i] >= 0:
                self.children[self.parents[i]].append(i)
        self.depth = np.zeros(self.n, np.int64)
        for i in self._topdown(np.nonzero(self.parents < 0)[0], strict=False):
            for c in self.children[i]:
                self.depth[c] = self.depth[i] + 1
        self.table = None

    def _topdown(self, nodes, strict):
        """nodes (and their descendants), parents before children"""
        out, stack = [], list(int(x) for x in nodes)
        seen = set()
        while stack:
            e = stack.pop()
            if e in seen:
                continue
            seen.add(e)
            out.append(e)
            stack.extend(self.children[e])
        if strict:
            out = [e for e in out if e not in set(int(x) for x in nodes)]
        return out

    def _recompose(self, nodes):
        nodes = np.array(sorted(set(int(x) for x in nodes if self.parents[x] >= 0)), np.int64)
        if not len(nodes):
            return
        d = self.depth[nodes]
        for lvl in np.unique(d):
            idx = nodes[d == lvl]
            self.G[idx] = _t(self.o.transform_compose(_b(self.G[self.parents[idx]]), _b(self.L[idx])))

    def set_table(self, attached, parent, system, instance, bone, rel):
        self.table = dict(A=np.asarray(attached, np.int64), P=np.asarray(parent, np.int64), S=np.asarray(system, np.int64),
                          I=np.asarray(instance, np.int64), B=np.asarray(bone, np.int64), R=np.asarray(rel, np.float32).reshape(-1, 7))
        self.rounds = table_rounds(self.parents, self.table["A"], self.table["P"]) if len(attached) else np.zeros(0, np.int64)

    def frame(self, poses, posed, local_edits=(), root_edits=()):
        """poses[s] = (pos [inst, bone, 3], rot [inst, bone, 4]); posed[s] bool.  -> moved mask per node."""
        marked = []
        for nodes, vals in local_edits:
            self.L[nodes] = vals
            marked += list(nodes)
        for nodes, vals in root_edits:
            self.G[nodes] = vals
            marked += list(nodes)
        closure = self._topdown(marked, strict=False)
        self._recompose(closure)
        moved = np.zeros(self.n, bool)
        moved[closure] = True
        t = self.table
        if t is None or not len(t["A"]):
            return moved
        for r in range(1, int(self.rounds.max()) + 1):
            ks = np.nonzero(self.rounds == r)[0]
            act = np.array([bool(posed[t["S"][k]]) or (moved[t["P"][k]] and self.entity[t["P"][k]] >= 0) for k in ks], bool)
            ks = ks[act]
            if not len(ks):
                continue
            A, P = t["A"][ks], t["P"][ks]
            bone7 = np.zeros((len(ks), 7), np.float32)
            for j, k in enumerate(ks):
                pos, rot = poses[t["S"][k]]
                bone7[j, :3] = pos[t["I"][k], t["B"][k]]
                bone7[j, 3:] = rot[t["I"][k], t["B"][k]]
            scale = np.ascontiguousarray(self.G["scale"][A])
            self.G[A] = _t(self.o.bone_attachments(_b(self.G[P]), bone7, t["R"][ks], scale))
            nr = A[self.parents[A] >= 0]
            if len(nr):
                self.L[nr] = _t(self.o.transform_compute_local(_b(self.G[self.parents[nr]]), _b(self.G[nr])))
            moved[A] = True
            sub = self._topdown(A, strict=True)
            self._recompose(sub)
            moved[sub] = True
        return moved


def _systems(ctx, specs, seed=2):
    """[(AnimationSystem, (pos, rot))] for (bones, instances) specs, posed once"""
    out = []
    for j, (bones, inst) in enumerate(specs):
        skel = scenes.skeleton(bones, seed=seed + j)
        clips = [scenes.clip(skel, frames=30, seed=s + 10 * j) for s in (3, 4)]
        a = lb.AnimationSystem(ctx, skel, clips, None, max_instances=inst)
        ci, tt = scenes.instance_times(inst, clips, seed=seed + j)
        a.setInstances(ci, tt)
        a.update(1.0 / 60.0, lb.PALETTE_POSE)
        out.append([a, a.getPose()])
    return out


def _step(systems, which):
    for j in which:
        systems[j][0].update(1.0 / 60.0, lb.PALETTE_POSE)
        systems[j][1] = systems[j][0].getPose()


def _table(rng, attached, parent, systems):
    m = len(attached)
    slot = rng.integers(0, len(systems), m)
    inst = np.array([rng.integers(0, systems[s][0].n) for s in slot], np.int64)
    bone = np.array([rng.integers(0, systems[s][0].skeleton.bone_count) for s in slot], np.int64)
    rel = np.concatenate([(rng.normal(size=(m, 3)) * 0.5).astype(np.float32), scenes.random_unit_quats(rng, m)], axis=1).astype(np.float32)
    return [np.asarray(attached), np.asarray(parent), slot, inst, bone, rel]


class Rig:
    """A library hierarchy and its oracle twin, driven frame by frame and compared after each."""

    def __init__(self, ctx, oracle, parents, seed, entity=None):
        rng = np.random.default_rng(seed)
        n = len(parents)
        self.ctx, self.rng = ctx, rng
        self.locals_ = _random_transforms(rng, n, 10.0)
        self.roots = _random_transforms(rng, n, 2000.0)
        self.entity = np.arange(n, dtype=np.int32) if entity is None else np.asarray(entity, np.int32)
        self.h = lb.Hierarchy(ctx, parents)
        self.h.setLocalTransforms(self.locals_)
        self.h.setRootTransforms(self.roots)
        self.h.setEntities(self.entity)
        self.h.propagate()
        self.w = AttachedWorld(oracle, parents, self.locals_, self.roots, self.entity)
        self.parents = np.asarray(parents)

    def set_table(self, table):
        self.h.setAttachments(*table)
        self.w.set_table(*table)

    def frame(self, systems, posed=None, local_nodes=(), root_nodes=(), what=""):
        rng = self.rng
        le, re_ = [], []
        if len(local_nodes):
            v = _random_transforms(rng, len(local_nodes), 10.0)
            self.h.setSubset(local_nodes, v)
            le.append((np.asarray(local_nodes), v))
        if len(root_nodes):
            v = _random_transforms(rng, len(root_nodes), 2000.0)
            self.h.setSubset(root_nodes, v, globals_=True)
            re_.append((np.asarray(root_nodes), v))
        ml = self.h.propagateAttached([s[0] for s in systems], posed)
        p = [True] * len(systems) if posed is None else list(posed)
        moved = self.w.frame([s[1] for s in systems], p, le, re_)
        self.check(ml, moved, what)
        return ml, moved

    def check(self, ml, moved, what):
        g = self.h.getTransforms()
        _bits_equal(g, self.w.G, f"{what}: globals")
        _bits_equal(self.h.getLocalTransforms(), self.w.L, f"{what}: locals")
        nodes = np.nonzero(moved & (self.entity >= 0))[0]
        assert ml.count == len(nodes), f"{what}: {ml.count} listed, the oracle moved {len(nodes)}"
        if len(nodes):
            ent = self.ctx.copy_to_host(ml.entities, ml.count, np.int32)
            tr = self.ctx.copy_to_host(ml.transforms, ml.count, lb.TRANSFORM_DTYPE)
            assert np.array_equal(ent, self.entity[nodes]), f"{what}: moved list"
            _bits_equal(tr, self.w.G[nodes], f"{what}: listed transforms")

    def rounds(self):
        r, nr = self.h.attachmentRounds()
        assert np.array_equal(r, self.w.rounds) and nr == int(self.w.rounds.max()), "attachment rounds"
        return r

    def close(self):
        self.h.close()


def _subtree(parents, x):
    ch = {}
    for i, p in enumerate(parents):
        ch.setdefault(int(p), []).append(i)
    out, st = [], [int(x)]
    while st:
        e = st.pop()
        out.append(e)
        st.extend(ch.get(e, []))
    return out


def _tree_of(parents, i):
    while parents[i] >= 0:
        i = int(parents[i])
    return i


# ------------------------------------------------------------------------------------------------------------------------ 1: one round
def test_one_round_on_a_forest(ctx, oracle):
    """Attached roots, attached non-roots and attached nodes with deep subtrees, each in its own tree, parents in trees without attachments:
    one round.  Posed frames, frames with edits only, a frame with root moves under attachment parents."""
    parents, _, _ = scenes.hierarchy_forest(20_000, 5, 3, seed=5)
    rig = Rig(ctx, oracle, parents, seed=1)
    rng = rig.rng
    systems = _systems(ctx, [(40, 200)])
    roots = np.nonzero(parents < 0)[0]
    trees = rng.permutation(roots[np.isin(roots, parents)])  # roots with children
    att_trees, par_trees = trees[: len(trees) // 2], trees[len(trees) // 2:]
    attached = []
    for j, t in enumerate(att_trees):
        sub = _subtree(parents, t)
        attached.append(t if j % 3 == 0 else sub[1 + (j * 7) % (len(sub) - 1)] if j % 3 == 1 else sub[1])  # root / any / level-1 (deep subtree)
    parent = [int(rng.choice(_subtree(parents, par_trees[j % len(par_trees)]))) for j in range(len(attached))]
    rig.set_table(_table(rng, attached, parent, systems))
    rig.frame(systems, what="first posed frame")
    assert (rig.rounds() == 1).all()
    _step(systems, [0])
    rig.frame(systems, local_nodes=rng.choice(np.nonzero(parents >= 0)[0], 50, replace=False), what="posed + local edits")
    rig.frame(systems, posed=[False], root_nodes=np.asarray(par_trees[:20]), what="parents' trees moved, nothing posed")
    rig.frame(systems, posed=[False], root_nodes=np.asarray(att_trees[:20]), what="attached trees moved, nothing posed")
    # the attached non-roots of moved trees take their new global scale into their attachment
    rig.frame(systems, root_nodes=np.asarray(att_trees[20:40]), what="attached trees moved, posed")
    rig.close()
    systems[0][0].close()


# ------------------------------------------------------------------------------------------------------------------------ 2: chains
@pytest.mark.parametrize("length", [2, 3, 8])
def test_chains_of_attachments(ctx, oracle, length):
    """horse -> rider -> sword: X_{j+1}'s parent node lies in X_j's attached subtree; plus, per chain, an attachment whose attached node
    lies inside another attached subtree.  Rounds reported = the order's rounds; a move of the first parent carries the whole chain."""
    parents, _, _ = scenes.hierarchy_forest(6000, 4, 3, seed=7)
    rig = Rig(ctx, oracle, parents, seed=2)
    rng = rig.rng
    systems = _systems(ctx, [(30, 64)])
    roots = rng.permutation(np.nonzero(parents < 0)[0])
    attached, parent = [], []
    chains = 12
    for c in range(chains):
        trees = roots[c * (length + 2):(c + 1) * (length + 2)]
        prev_tree = trees[0]
        for j in range(length):
            sub_prev = _subtree(parents, prev_tree)
            parent.append(int(sub_prev[min(len(sub_prev) - 1, 1 + j)]))  # inside the previous attached subtree (or the horse's tree)
            attached.append(int(trees[j + 1]))
            prev_tree = trees[j + 1]
        # an attached node inside the first rider's subtree, following a bone of an unrelated tree
        attached.append(int(_subtree(parents, trees[1])[-1]))  # a leaf below the first rider
        parent.append(int(rng.choice(_subtree(parents, trees[length + 1]))))
    rig.set_table(_table(rng, attached, parent, systems))
    rig.frame(systems, what="posed")
    r = rig.rounds()
    assert r.max() == length
    horses = [int(_tree_of(parents, parent[c * (length + 1)])) for c in range(chains)]
    rig.frame(systems, posed=[False], root_nodes=np.asarray(horses[: chains // 2]), what="horses moved")
    rig.frame(systems, posed=[False], what="nothing")
    _step(systems, [0])
    rig.frame(systems, root_nodes=np.asarray(horses[chains // 2:]), what="posed + horses moved")
    rig.close()
    systems[0][0].close()


# ------------------------------------------------------------------------------------------------------------------------ 3: pins
def test_pins_keep_attached_globals(ctx, oracle):
    """A frame with nothing posed or moved leaves every global as it was, while plain propagate on the same scene recomposes some attached
    non-root from its computed local to another value; a moved world parent of an inactive attachment leaves its node at W.compose(local)."""
    parents, _, _ = scenes.hierarchy_forest(30_000, 5, 4, seed=9)
    rig = Rig(ctx, oracle, parents, seed=3)
    rng = rig.rng
    systems = _systems(ctx, [(40, 100)])
    roots = np.nonzero(parents < 0)[0]
    half = len(roots) // 2
    cand = np.nonzero((parents >= 0))[0]
    cand = cand[np.isin([_tree_of(parents, i) for i in cand], roots[:half])]
    attached = rng.choice(cand, 1500, replace=False)
    # no attached node below another: one round, and every attached node's world parent is unattached
    keep, taken = [], set()
    for a in attached:
        chain = [int(a)]
        while parents[chain[-1]] >= 0:
            chain.append(int(parents[chain[-1]]))
        if not taken.intersection(chain):
            keep.append(int(a))
            taken.update(chain)
    attached = np.array(keep)
    parent = rng.choice(np.nonzero(np.isin([_tree_of(parents, i) for i in range(len(parents))], roots[half:]))[0], len(attached))
    rig.set_table(_table(rng, attached, parent, systems))
    rig.frame(systems, what="posed")
    before = rig.h.getTransforms()
    ml, _ = rig.frame(systems, posed=[False], what="nothing posed or moved")
    assert ml.count == 0
    _bits_equal(rig.h.getTransforms(), before, "nothing posed or moved")
    twin = lb.Hierarchy(ctx, parents)
    twin.setLocalTransforms(rig.h.getLocalTransforms())
    twin.setTransforms(before)
    twin.propagate()
    after = twin.getTransforms()
    drift = [f for f in FIELDS if after[f][attached].tobytes() != before[f][attached].tobytes()]
    assert drift, "plain propagate recomposes the attached nodes to the same bits: the pins are not exercised"
    twin.close()
    # the world parent of an attached node moves; its attachment's parent neither moves nor is posed
    w = np.array([int(parents[a]) for a in attached[:40]])
    ml, moved = rig.frame(systems, posed=[False], local_nodes=w, what="world parents moved")
    g = rig.h.getTransforms()
    l = rig.h.getLocalTransforms()
    exp = _t(oracle.transform_compose(_b(g[w]), _b(l[attached[:40]])))
    _bits_equal(g[attached[:40]], exp, "inactive attachment under a moved world parent")
    rig.close()
    systems[0][0].close()


# ------------------------------------------------------------------------------------------------------------------------ 4 + 5: activity
def test_activity_and_two_systems(ctx, oracle):
    """posed per system (two systems with 40 and 90 bones in one call), a parent whose entity id is -1 does not trigger, a parent moved by
    an earlier round does."""
    parents, _, _ = scenes.hierarchy_forest(8000, 4, 3, seed=11)
    n = len(parents)
    rng = np.random.default_rng(4)
    entity = np.where(rng.random(n) < 0.75, np.arange(n), -1).astype(np.int32)
    rig = Rig(ctx, oracle, parents, seed=4, entity=entity)
    systems = _systems(ctx, [(40, 50), (90, 30)])
    roots = rng.permutation(np.nonzero(parents < 0)[0])
    attached, parent = [], []
    for j in range(0, 120, 3):
        t0, t1, t2 = roots[j:j + 3]
        attached += [int(t1), int(t2)]
        parent += [int(rng.choice(_subtree(parents, t0))), int(rng.choice(_subtree(parents, t1)))]  # the second follows the first's subtree
    tab = _table(rng, attached, parent, systems)
    rig.set_table(tab)
    rig.frame(systems, what="both posed")
    assert rig.rounds().max() == 2
    for posed in ([True, False], [False, True]):
        _step(systems, [posed.index(True)])
        rig.frame(systems, posed=posed, what=f"posed {posed}")
    first = np.array(parent[0::2])
    silent = first[entity[first] < 0]
    loud = first[entity[first] >= 0]
    assert len(silent) and len(loud)
    horses = np.array([_tree_of(parents, p) for p in first])
    rig.frame(systems, posed=[False, False], root_nodes=np.unique(horses), what="parents moved, some without a listener")
    rig.close()
    for s in systems:
        s[0].close()


# ------------------------------------------------------------------------------------------------------------------------ 6: launch shapes
def _chain(depth, width):
    p = np.full(depth * width, -1, np.int32)
    p[width:] = np.arange(width * (depth - 1), dtype=np.int32)
    return p


def _star(children, extra_roots):
    p = np.full(children + 1 + extra_roots, -1, np.int32)
    p[1:children + 1] = 0
    return p


@pytest.mark.parametrize("shape", ["chain_300", "star_8193"])
def test_launch_shapes(ctx, oracle, shape):
    """A 300-deep chain (recomposes past the small-levels kernel's 30 levels) and an 8193-child star (the per-level kernel), with rounds
    whose attachments are all inactive."""
    rng = np.random.default_rng(5)
    if shape == "chain_300":
        parents = _chain(300, 4)  # chain c: nodes c, c + 4, ...
        attached = [4 * 5 + 1, 4 * 200 + 2, 4 * 250 + 1]  # chain 1 at depth 5 follows chain 0, chain 2 follows chain 1 deep down, ...
        parent = [4 * 10 + 0, 4 * 100 + 1, 4 * 280 + 3]
    else:
        parents = _star(8193, 40)
        attached = [0, 5, 8196, 8197]  # the star's root (its 8193 children recomposed), one of its children, two single roots
        parent = [8194, 8196, 8195, 8196]
    rig = Rig(ctx, oracle, parents, seed=6)
    systems = _systems(ctx, [(20, 8)])
    rig.set_table(_table(rng, attached, parent, systems))
    rig.frame(systems, what=f"{shape}: posed")
    assert rig.rounds().max() >= 2
    rig.frame(systems, posed=[False], what=f"{shape}: nothing active")
    src = [int(_tree_of(parents, parent[0]))]
    rig.frame(systems, posed=[False], root_nodes=np.asarray(src), what=f"{shape}: first parent's root moved")
    rig.frame(systems, posed=[False], local_nodes=np.asarray([attached[0]]), what=f"{shape}: an attached node's local written")
    rig.close()
    systems[0][0].close()


def test_empty_table_is_propagate_moved(ctx, oracle):
    parents, _, _ = scenes.hierarchy_forest(5000, 5, 3, seed=12)
    a = Rig(ctx, oracle, parents, seed=7)
    b = Rig(ctx, oracle, parents, seed=7)
    systems = _systems(ctx, [(20, 8)])
    unposed = lb.AnimationSystem(ctx, scenes.skeleton(20), [scenes.clip(scenes.skeleton(20), frames=10)], None, max_instances=4)
    rng = np.random.default_rng(1)
    for k in range(3):
        nodes = rng.choice(len(parents), 40, replace=False).astype(np.uint32)
        vals = _random_transforms(rng, 40, 10.0)
        for x in (a, b):
            x.h.setSubset(nodes, vals)
        ma = a.h.propagateAttached([[], [s[0] for s in systems], [unposed]][k])  # an empty table does not look at the systems
        mb = b.h.propagateMoved()
        assert ma.count == mb.count
        _bits_equal(a.h.getTransforms(), b.h.getTransforms(), "empty table")
        assert ctx.copy_to_host(ma.entities, ma.count, np.int32).tobytes() == ctx.copy_to_host(mb.entities, mb.count, np.int32).tobytes()
    a.close()
    b.close()
    systems[0][0].close()
    unposed.close()


# ------------------------------------------------------------------------------------------------------------------------ 7: refusals
def _state(h):
    return h.getTransforms(), h.getLocalTransforms()


def _same(h, st, what):
    g, l = _state(h)
    _bits_equal(g, st[0], f"{what}: globals")
    _bits_equal(l, st[1], f"{what}: locals")


def _refused(code, fn):
    with pytest.raises(LumixB200Error) as e:
        fn()
    assert e.value.code == code, str(e.value)


def test_refusals_leave_the_hierarchy_as_it_was(ctx, oracle):
    parents, _, _ = scenes.hierarchy_forest(3000, 4, 3, seed=13)
    n = len(parents)
    rig = Rig(ctx, oracle, parents, seed=8)
    rng = rig.rng
    systems = _systems(ctx, [(30, 16), (50, 8)])
    other_ctx = lb.Context(0)
    foreign = _systems(other_ctx, [(30, 16)])
    unposed = lb.AnimationSystem(ctx, scenes.skeleton(30), [scenes.clip(scenes.skeleton(30), frames=10)], None, max_instances=4)
    roots = rng.permutation(np.nonzero(parents < 0)[0])
    attached = [int(roots[1]), int(roots[2])]
    parent = [int(_subtree(parents, roots[0])[3]), int(_subtree(parents, roots[1])[2])]
    tab = _table(rng, attached, parent, systems)
    tab[2][:] = [0, 1]
    tab[3][:] = [3, 2]
    tab[4][:] = [7, 9]
    rig.set_table(tab)
    rig.frame(systems, what="posed")
    h = rig.h
    # marks stay: an edit before every refusal must still be listed afterwards
    x = int(np.nonzero(parents >= 0)[0][5])
    h.markMoved([x])
    st = _state(h)
    live = [s[0] for s in systems]
    t = [c.copy() for c in tab]
    t[0][0] = n
    _refused(ERR_INVALID, lambda: h.setAttachments(*t))
    t = [c.copy() for c in tab]
    t[1][0] = n
    _refused(ERR_INVALID, lambda: h.setAttachments(*t))
    t = [c.copy() for c in tab]
    t[1][0] = t[0][0]
    _refused(ERR_INVALID, lambda: h.setAttachments(*t))
    t = [c.copy() for c in tab]
    t[0][1] = t[0][0]
    _refused(ERR_INVALID, lambda: h.setAttachments(*t))
    _refused(ERR_INVALID, lambda: h.propagateAttached(live[:1]))                      # slot 1 >= 1 system
    t = [c.copy() for c in tab]
    t[2][1] = 0xFFFFFFFF  # a slot no call can have: accepted by set_attachments (it has no systems), refused by every call
    h.setAttachments(*t)
    _refused(ERR_INVALID, lambda: h.propagateAttached(live))
    h.setAttachments(*tab)
    _refused(ERR_STATE, lambda: h.propagateAttached([live[0], unposed]))               # no absolute poses
    _refused(ERR_STATE, lambda: h.propagateAttached([foreign[0][0], live[1]]))         # another context
    out = lb.hierarchy._Moved()
    arr = (C.c_void_p * 2)(live[0].h, None)
    assert h.L.lb200_hierarchy_propagate_attached(h.h, arr, None, C.c_uint32(2), None, C.byref(out), None) == ERR_STATE  # a NULL system
    small = _systems(ctx, [(7, 16), (50, 2)])
    _refused(ERR_INVALID, lambda: h.propagateAttached([small[0][0], live[1]]))         # bone 7 >= 8 bones
    _refused(ERR_INVALID, lambda: h.propagateAttached([live[0], small[1][0]]))         # instance 2 >= 2 instances
    _same(h, st, "after the refusals")
    # a cycle: the first attached tree's node becomes the parent of its own parent's tree
    t = [c.copy() for c in tab]
    t[1][1] = int(_subtree(parents, roots[0])[1])  # X1 follows roots[0]'s tree, X0 attaches roots[1] to roots[0]'s tree: fine
    t[1][0] = int(_subtree(parents, roots[1])[1])  # X0 follows a node below its own attached node: a cycle
    h.setAttachments(*t)
    _refused(ERR_INVALID, lambda: h.propagateAttached(live))
    _same(h, st, "after the cycle")
    h.setAttachments(*tab)
    # a cycle created by set_parents: roots[0] moves below roots[1]'s subtree (X0 attaches roots[1] to roots[0]'s tree)
    p2 = parents.copy()
    p2[roots[0]] = int(_subtree(parents, roots[1])[1])
    h.setParents(p2)
    _refused(ERR_INVALID, lambda: h.propagateAttached(live))
    _same(h, st, "after the re-parenting cycle")
    h.setParents(parents)
    ml = h.propagateAttached(live, posed=[False, False])
    ent = ctx.copy_to_host(ml.entities, ml.count, np.int32)
    assert x in set(ent.tolist()), "the mark made before the refusals is still there"
    # a shrink below a table node: refused until the table is set again, then a table inside the hierarchy runs
    keep = max(attached + parent)
    p3 = np.where(parents[:keep] < keep, parents[:keep], -1).astype(np.int32)
    h.setParents(p3)
    before = h.getTransforms()
    h.markMoved([0])
    _refused(ERR_STATE, lambda: h.propagateAttached(live))
    _bits_equal(h.getTransforms(), before, "after the shrink")
    small_tab = [c[:1].copy() for c in tab]
    r3 = np.nonzero(p3 < 0)[0]
    small_tab[0][0], small_tab[1][0] = r3[0], r3[1]  # one root follows a bone of another root
    h.setAttachments(*small_tab)
    ml = h.propagateAttached(live, posed=[False, False])
    assert ml.count >= 1, "the mark made before the refused call is listed"
    rig.close()
    for s in systems + small:
        s[0].close()
    unposed.close()
    foreign[0][0].close()
    other_ctx.close()


# ------------------------------------------------------------------------------------------------------------------------ 8: device chain
LIGHT = (0.3, -0.8, 0.2)
CASCADES = (40.0, 200.0, 900.0, 2500.0)
SHADOW_BUCKETS = [0, 0xff, 0xff, 1]


def _canon(keys, values):
    o = np.lexsort((values, keys))
    return keys[o], values[o]


def _compare_view(got, exp, what):
    gk, gv = _canon(got["keys"], got["values"])
    ek, ev = _canon(exp["keys"], exp["values"])
    assert np.array_equal(gk, ek) and np.array_equal(gv, ev), f"{what}: pairs differ ({len(gk)} against {len(ek)})"
    assert np.array_equal(got["group_count"], exp["group_count"]) and np.array_equal(got["group_offset"], exp["group_offset"]), what
    go, eo = np.argsort(got["group_renderables"], kind="stable"), np.argsort(exp["group_renderables"], kind="stable")
    assert np.array_equal(got["group_renderables"][go], exp["group_renderables"][eo]), what
    assert np.array_equal(got["instance_data"][go], exp["instance_data"][eo]), what


def test_device_chain_with_attachments(ctx, oracle):
    """Edits plus posed instances -> propagateAttached -> moveDevice(list) -> set_many_device(list) -> cull_views -> createSortKeysViews
    -> endFrame over three frames, against the oracle frame in which exactly the moved list is MOVED and re-set."""
    parents, _, _ = scenes.hierarchy_forest(200_000, 4, 5, seed=3, root_extent=(2500.0, 300.0, 2500.0))
    n = len(parents)
    rng = np.random.default_rng(17)
    entity = rng.permutation(n).astype(np.int32)
    rig = Rig(ctx, oracle, parents, seed=9, entity=entity)
    rig.roots["pos"] = (rng.random((n, 3)) * 2.0 - 1.0) * np.array([2500.0, 300.0, 2500.0])
    rig.h.setRootTransforms(rig.roots)
    rig.h.propagate()
    rig.w = AttachedWorld(oracle, parents, rig.locals_, rig.roots, entity)
    systems = _systems(ctx, [(40, 500)])
    roots = np.nonzero(parents < 0)[0]
    roots = rng.permutation(roots[np.isin(roots, parents)])  # roots with children
    m = 200
    attached = [int(r) for r in roots[:m]] + [int(_subtree(parents, r)[1]) for r in roots[m:2 * m]]
    parent = [int(rng.choice(_subtree(parents, r))) for r in roots[2 * m:4 * m]]
    rig.set_table(_table(rng, attached, parent, systems))
    br = (0.5 + 2.5 * rng.random(n)).astype(np.float32)
    g = rig.w.G
    tr_e = np.zeros(n, lb.TRANSFORM_DTYPE)
    tr_e[entity] = g
    pos_e = np.zeros((n, 3))
    pos_e[entity] = g["pos"]
    rad_e = np.zeros(n, np.float32)
    rad_e[entity] = oracle.sphere_radius(_b(g), br)
    types = np.zeros(n, np.uint8)
    ents = np.arange(n, dtype=np.int32)
    cs = lb.CullingSystem(ctx)
    cs.add(ents, types, pos_e, rad_e)
    cs.set_replicas(1)
    oc = oracle.OracleCulling()
    oc.add(ents, types, pos_e, rad_e)
    sk = scenes.sortkey_setup(n, types, pos_e, seed=23, moved_fraction=0.0)
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=4 * n, max_instances=4 * n)
    S.setModels(sk["models"], sk["meshes"])
    S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(tr_e)
    lod, pf = sk["lod"].copy(), sk["pose_frame"].copy()
    prev_exp = np.zeros(n, lb.TRANSFORM_DTYPE)
    cam = dict(scenes.c1_frustum_args(), far=2500.0)
    args = [cam] + scenes.shadow_cascade_args(cam, LIGHT, CASCADES)
    frusta = [lb.frustum_perspective(**a) if "fov" in a else lb.frustum_ortho(**a) for a in args]
    for frame in range(3):
        _step(systems, [0])
        moved_roots = rng.choice(roots[4 * m:], 200, replace=False).astype(np.uint32)
        if frame == 2:
            moved_roots = np.union1d(moved_roots, [_tree_of(parents, p) for p in parent[:50]]).astype(np.uint32)
        vals = rig.roots[moved_roots].copy()
        vals["pos"] += rng.normal(size=(len(moved_roots), 3)) * 400.0
        vals["rot"] = scenes.random_unit_quats(rng, len(moved_roots))
        rig.roots[moved_roots] = vals
        rig.h.setSubset(moved_roots, vals, globals_=True)
        posed = [frame != 1]
        ml = rig.h.propagateAttached([systems[0][0]], posed, br if frame == 0 else None)
        moved = rig.w.frame([systems[0][1]], posed, (), [(moved_roots, vals)])
        rig.check(ml, moved, f"frame {frame}")
        S.moveDevice(ml.entities, ml.transforms, ml.count)
        cs.set_many_device(ml.pos3, ml.radius, ml.count, dev_entities=ml.entities, max_entity=n - 1)
        cs.cull_views(frusta, want_counts=False)
        views = [sortkeys.make_view(a["position"], cam["position"], 0.15, 1.25, 50 + frame, k > 0, sk["max_sort_key"],
                                    *((sk["layer_to_bucket"], sk["depth_sorted_buckets"]) if k == 0 else (SHADOW_BUCKETS, ())))
                 for k, a in enumerate(args)]
        res = S.createSortKeysViews(cs, views)
        got = [S.readView(k, r) for k, r in enumerate(res)]
        S.endFrame()
        prev = S.prevTransforms()
        nodes = np.nonzero(moved)[0]
        ce = entity[nodes]
        g = rig.w.G
        new_pos = np.ascontiguousarray(g["pos"][nodes])
        new_rad = oracle.sphere_radius(_b(g[nodes]), br[nodes])
        oc.set(ce, new_pos, new_rad)
        tr_e[ce] = g[nodes]
        flags = sk["flags"].copy()
        flags[ce] |= sortkeys.MOVED
        for v, (f, view) in enumerate(zip(frusta, views)):
            oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f))
            exp = oracle.create_sort_keys(oids, otys, tr_e, sk["model_of"], lod, flags, pf, sk["decal_sort_key"], sk["decal_layer"],
                                          sk["models"], sk["meshes"], view)
            assert res[v].n_keys == len(exp["keys"]), f"frame {frame} view {v}"
            _compare_view(got[v], exp, f"frame {frame} view {v}")
        prev_exp[ce] = tr_e[ce]
        _bits_equal(prev, prev_exp, f"frame {frame}: prev_frame_transform")
    S.close()
    cs.close()
    rig.close()
    systems[0][0].close()


# ------------------------------------------------------------------------------------------------------------------------ reference World
SHIM = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libengine_shim_b200.so")


@pytest.fixture(scope="module")
def shim(oracle):
    if not os.path.exists(SHIM) or not oracle.ref_available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    L = C.CDLL(SHIM)
    os.environ["LB200_ENGINE_SHIM_LOADED"] = "1"  # the engine's job system cannot be shut down on Linux: tests/conftest.py leaves with os._exit
    L.wshim_run.restype = C.c_int
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class RefWorld:
    """The reference's own World (oracle/_ref/libengine_shim_b200.so, wshim_run) kept across frames by replay: every call builds the World
    from the same parents, locals and root globals and applies every World::setTransform made so far, in order.  A frame's attachments are
    evaluated round by round with the reference's own updateBoneAttachment arithmetic (oracle.bone_attachments(use_ref=True)) on the World's
    globals and applied with setTransform; an attachment runs when its system is posed or its parent fired `transformed` in this frame."""

    def __init__(self, shim, oracle, parents, locals_, roots, listens):
        self.shim, self.o = shim, oracle
        self.parents, self.locals_, self.roots, self.listens = parents, np.ascontiguousarray(locals_), np.ascontiguousarray(roots), listens
        self.ops = []
        self.G, self.L, self.calls = self.run([])

    def run(self, ops):
        n = len(self.parents)
        moved = np.array([e for e, _ in ops], np.uint32)
        vals = np.zeros(len(ops), lb.TRANSFORM_DTYPE)
        for k, (_, v) in enumerate(ops):
            vals[k] = v
        out_ref, out_b, out_l = (np.zeros(n, lb.TRANSFORM_DTYPE) for _ in range(3))
        calls_ref, calls_b = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        seconds = np.zeros(2)
        rc = self.shim.wshim_run(_p(self.parents), _p(self.locals_), _p(self.roots), C.c_uint32(n), _p(self.listens),
                                 _p(moved) if len(ops) else None, _p(vals) if len(ops) else None, C.c_uint32(len(ops)), C.c_uint32(1), C.c_int(0),
                                 _p(out_ref), _p(out_b), _p(calls_ref), _p(calls_b), _p(seconds), _p(out_l))
        assert rc == 0
        return out_ref, out_l, calls_ref

    def frame(self, table, rounds, poses, posed, root_edits):
        """-> (globals, locals, entities whose `transformed` fired in this frame)"""
        base = self.calls
        ops = self.ops + [(int(e), v) for e, v in zip(*root_edits)]
        G, L, calls = self.run(ops)
        for r in range(1, int(rounds.max()) + 1):
            fired = calls > base
            ks = [k for k in np.nonzero(rounds == r)[0] if posed[table[2][k]] or fired[table[1][k]]]
            if not ks:
                continue
            A, P = table[0][ks].astype(np.int64), table[1][ks].astype(np.int64)
            bone7 = np.array([np.concatenate([poses[table[2][k]][0][table[3][k], table[4][k]], poses[table[2][k]][1][table[3][k], table[4][k]]]) for k in ks],
                             np.float32)
            vals = _t(self.o.bone_attachments(_b(G[P]), bone7, table[5][ks], np.ascontiguousarray(G["scale"][A]), use_ref=True))
            ops += [(int(a), v) for a, v in zip(A, vals)]
            G, L, calls = self.run(ops)
        self.ops, self.G, self.L = ops, G, L
        fired = calls > base
        self.calls = calls
        return G, L, fired


@pytest.mark.parametrize("scene", ["forest", "chain", "pins"])
def test_frames_match_the_reference_world(ctx, oracle, shim, scene):
    """The same frames through the library and through the reference's own World::setTransform, round by round: the moved list is exactly
    the set of entities whose `transformed` delegates the World fired (the edits' subtrees, the attached nodes and their subtrees, the
    activity rule with listeners).  Transforms are not compared here: the World recomposes a node only when it moves, from the local
    transformEntity(update_local) recomputed from its global, while every propagate recomposes every unpinned node from its local, and
    compose o computeLocal does not settle, so the two states part on nodes no attachment touches.  The frames' transforms are held bit
    for bit to AttachedWorld above."""
    parents, locals_, roots = scenes.hierarchy_forest(4000, 4, 3, seed=21)
    n = len(parents)
    rng = np.random.default_rng(31)
    listens = (rng.random(n) < 0.85).astype(np.uint8)
    entity = np.where(listens == 1, np.arange(n), -1).astype(np.int32)
    ref = RefWorld(shim, oracle, parents, locals_, roots, listens)
    h = lb.Hierarchy(ctx, parents)
    h.setEntities(entity)
    h.setTransforms(ref.G)
    h.computeLocalTransforms()
    nonroot = parents >= 0
    _bits_equal(h.getLocalTransforms()[nonroot], ref.L[nonroot], "the World's locals")
    systems = _systems(ctx, [(30, 32)])
    tree_roots = rng.permutation(np.nonzero(parents < 0)[0])
    if scene == "forest":    # attached roots and attached inner nodes with subtrees, one round
        attached = [int(r) if j % 2 else int(_subtree(parents, r)[1]) for j, r in enumerate(tree_roots[:20])]
        parent = [int(rng.choice(_subtree(parents, r))) for r in tree_roots[20:40]]
    elif scene == "chain":   # horse -> rider -> sword, and a node inside the rider's subtree
        attached, parent = [], []
        for c in range(6):
            t = tree_roots[5 * c:5 * c + 5]
            attached += [int(t[1]), int(t[2]), int(_subtree(parents, t[1])[-1])]
            parent += [int(_subtree(parents, t[0])[3]), int(_subtree(parents, t[1])[2]), int(rng.choice(_subtree(parents, t[3])))]
    else:                    # attached inner nodes whose world parents move while their attachment parents stay
        attached = [int(_subtree(parents, r)[1]) for r in tree_roots[:20]]
        parent = [int(rng.choice(_subtree(parents, r))) for r in tree_roots[20:40]]
    table = _table(rng, attached, parent, systems)
    table = [np.asarray(table[0], np.uint32), np.asarray(table[1], np.uint32), np.asarray(table[2], np.int64), np.asarray(table[3], np.int64),
             np.asarray(table[4], np.int64), np.ascontiguousarray(table[5], np.float32)]
    h.setAttachments(*table)
    rounds = table_rounds(parents, table[0], table[1])
    own_trees = [_tree_of(parents, a) for a in attached]
    par_trees = [_tree_of(parents, p) for p in parent]
    frames = [("posed", None, [])]
    if scene == "pins":
        frames += [("nothing", [False], []), ("world parents moved", [False], own_trees[:10]), ("both moved", [False], own_trees[10:] + par_trees[10:])]
    else:
        frames += [("parents moved", [False], par_trees[: len(par_trees) // 2]), ("posed + attached trees moved", None, own_trees[::3])]
    for what, posed, moved_roots in frames:
        if posed is None:
            _step(systems, [0])
        moved_roots = np.unique(np.asarray(moved_roots, np.uint32))
        vals = _random_transforms(rng, len(moved_roots), 2000.0)
        if len(moved_roots):
            h.setSubset(moved_roots, vals, globals_=True)
        ml = h.propagateAttached([systems[0][0]], posed)
        _, _, fired = ref.frame(table, rounds, [systems[0][1]], [True] if posed is None else posed, (moved_roots, vals))
        ent = ctx.copy_to_host(ml.entities, ml.count, np.int32) if ml.count else np.zeros(0, np.int32)
        assert np.array_equal(np.sort(ent), np.nonzero(fired)[0]), f"{scene} / {what}: moved list against the World's delegates"
        if what == "nothing":
            assert ml.count == 0
    h.close()
    systems[0][0].close()
