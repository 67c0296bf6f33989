"""numpy restatement of mapping::PoseGraph3D's bookkeeping on the fork's live loop-closure path (pose_graph_3d.cc:67-144,
:335-399, :444-470, :718-770, :914-952; constraint_builder_3d.cc:162-259, :334), the counterpart of dl_pose_graph_3d_* in the
manner of schur_oracle.py. The two device stages are injected: `search(pairs)` returns one (found, zbar7, translation_weight,
rotation_weight) per (submap, node, guess) pair, `solve(submap_poses, node_poses, constraints, frozen)` returns the optimized
(submap_poses, node_poses). Poses are 7-vectors (t xyz, q wxyz); the formulas are those of the library's Rigid3 math
(rigid_transform.h: composition re-normalises, inverse conjugates)."""
import numpy as np

IDENTITY = np.array([0.0, 0, 0, 1, 0, 0, 0])
INTRA, INTER = 0, 1


def rotate(q, v):
    qv = np.asarray(q[1:], np.float64)
    uv = np.cross(qv, v)
    uv = uv + uv
    return v + q[0] * uv + np.cross(qv, uv)


def qmul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])


def compose(a, b):
    q = qmul(a[3:], b[3:])
    return np.concatenate([rotate(a[3:], b[:3]) + a[:3], q / np.linalg.norm(q)])


def inverse(a):
    qi = np.array([a[3], -a[4], -a[5], -a[6]])
    return np.concatenate([-rotate(qi, a[:3]), qi])


def yaw_quaternion(angle):
    return np.array([np.cos(0.5 * angle), 0.0, 0.0, np.sin(0.5 * angle)])


def get_yaw(q):
    d = rotate(q, np.array([1.0, 0.0, 0.0]))
    return np.arctan2(d[1], d[0])


def yaw_free_alignment(submap_pose):
    """Embed3D(Rigid2d::Rotation(-yaw)) * Rigid3d::Rotation(rotation) (constraint_builder_3d.cc:241-251)."""
    aligned = np.concatenate([[0.0, 0.0, 0.0], submap_pose[3:]])
    return compose(np.concatenate([[0.0, 0.0, 0.0], yaw_quaternion(-get_yaw(aligned[3:]))]), aligned)


def embed_2d(x, y, theta):
    return np.concatenate([[x, y, 0.0], yaw_quaternion(theta)])


def pose_guess(local_submap_from, local_submap_to, match_xytheta, local_node_pose):
    """T_G1_S1 * M2D * T_S2_G2 * node_pose_in_submap_from (constraint_builder_3d.cc:226-259), with the submaps' LOCAL poses."""
    t_g1_s1 = inverse(yaw_free_alignment(local_submap_to))
    t_s2_g2 = yaw_free_alignment(local_submap_from)
    left = compose(compose(t_g1_s1, embed_2d(*match_xytheta)), t_s2_g2)
    return compose(left, compose(inverse(local_submap_from), local_node_pose))


def match_from_truth(local_submap_from, local_submap_to, local_to_world_from, local_to_world_to):
    """The yaw-and-xy relation between the two yaw-free gravity-aligned submap frames that makes pose_guess exact when the
    submaps' local frames are placed in one world by local_to_world_*: (x, y, theta)."""
    rel = compose(inverse(compose(local_to_world_to, local_submap_to)), compose(local_to_world_from, local_submap_from))
    m = compose(compose(yaw_free_alignment(local_submap_to), rel), inverse(yaw_free_alignment(local_submap_from)))
    return m[0], m[1], get_yaw(m[3:])


class PoseGraph3D:
    def __init__(self, optimize_every_n_nodes, every_nodes_to_find_constraint, matcher_weights=(5e2, 1.6e3)):
        self.n_opt, self.every = optimize_every_n_nodes, every_nodes_to_find_constraint
        self.weights = matcher_weights
        self.submaps = {}        # trajectory -> list of dict(local, global, finished, node_ids, optimized)
        self.nodes = {}          # trajectory -> list of dict(local, global, problem_global)
        self.frozen = set()
        self.constraints = []    # (submap id, node id, zbar, tw, rw, tag)
        self.pending = []
        self.computed = {}       # submap id -> set of node ids
        self.since_last = 0
        self.searched = []       # every (submap id, node id, guess) handed to search, in order
        self.solves = []         # inputs of every solve: (submap ids, node ids, submap poses, node poses, constraints, frozen)

    def local_to_global(self, t, optimized=True):
        for s in reversed(self.submaps.get(t, [])):
            if not optimized or s["optimized"] is not None:
                return compose(s["optimized"] if optimized else s["global"], inverse(s["local"]))
        return IDENTITY.copy()

    def add_node(self, t, local_pose, insertion, matches=(), search=None, solve=None):
        """insertion: [(submap_index, finished, local_pose7)]; matches: [(trajectory, index, x, y, theta)] -> True if optimized."""
        local_pose = np.asarray(local_pose, np.float64)
        subs = self.submaps.setdefault(t, [])
        nodes = self.nodes.setdefault(t, [])
        S = len(subs)
        idx = [i for i, _, _ in insertion]
        if len(insertion) == 1:
            assert idx == [0] and S <= 1
            back_new = S == 0
        else:
            assert (S >= 1 and idx == [S - 1, S]) or (S >= 2 and idx == [S - 2, S - 1])
            back_new = idx[1] == S
        if matches:
            assert insertion[0][1]
        node_index = len(nodes)
        node = {"local": local_pose, "global": compose(self.local_to_global(t), local_pose)}     # AddNode (:115-116)
        if back_new:
            local = np.asarray(insertion[-1][2], np.float64)
            if len(insertion) == 1:    # InitializeGlobalSubmapPoses, one submap
                g = compose(self.local_to_global(t), local)
            else:                      # two submaps, the back one new
                f = subs[idx[0]]
                g = compose(compose(f["global"], inverse(f["local"])), local)
            subs.append({"local": local, "global": g, "finished": False, "node_ids": [], "optimized": None})
        m = subs[idx[0]]
        node["problem_global"] = compose(compose(m["global"], inverse(m["local"])), local_pose)
        nodes.append(node)
        for i in idx:
            subs[i]["node_ids"].append(node_index)
            self.constraints.append(((t, i), (t, node_index), compose(inverse(subs[i]["local"]), local_pose),
                                     self.weights[0], self.weights[1], INTRA))
        if insertion[0][1]:
            frm = subs[idx[0]]
            frm["finished"] = True
            pairs = []
            for mt in sorted(matches, key=lambda x: (x[0], x[1])):
                to = (mt[0], mt[1])
                target = self.submaps[to[0]][to[1]]
                assert target["finished"] and to != (t, idx[0])
                for j, n in enumerate(frm["node_ids"]):
                    if j % self.every != 0 or (t, n) in self.computed.get(to, set()):
                        continue
                    pairs.append((to, (t, n), pose_guess(frm["local"], target["local"], mt[2:], nodes[n]["local"])))
            self.searched.extend(pairs)
            if pairs:
                for (to, nid, _), (found, zbar, tw, rw) in zip(pairs, search(pairs)):
                    if found:
                        self.computed.setdefault(to, set()).add(nid)
                        self.pending.append((to, nid, np.asarray(zbar, np.float64), tw, rw, INTER))
        self.since_last += 1
        if self.n_opt > 0 and self.since_last > self.n_opt:
            self.optimize(solve)
            return True
        return False

    def optimize(self, solve):
        """HandleWorkQueue's dedup across tags, then Solve and RunOptimization's update."""
        for c in self.pending:
            if not any(c[0] == d[0] and c[1] == d[1] for d in self.constraints):
                self.constraints.append(c)
        self.pending = []
        sids = [(t, i) for t in sorted(self.submaps) for i in range(len(self.submaps[t]))]
        nids = [(t, i) for t in sorted(self.nodes) for i in range(len(self.nodes[t]))]
        if not sids:
            return
        sp = np.array([self.submaps[t][i]["global"] for t, i in sids])
        npo = np.array([self.nodes[t][i]["problem_global"] for t, i in nids])
        frozen = [t in self.frozen for t, _ in sids] + [t in self.frozen for t, _ in nids]
        si, ni = {s: k for k, s in enumerate(sids)}, {n: k for k, n in enumerate(nids)}
        cons = [(si[c[0]], ni[c[1]], c[2], c[3], c[4]) for c in self.constraints]
        self.solves.append((sids, nids, sp, npo, cons, frozen))
        sp, npo = solve(sp, npo, cons, frozen)
        for k, (t, i) in enumerate(sids):
            self.submaps[t][i]["global"] = np.asarray(sp[k])
        for k, (t, i) in enumerate(nids):
            self.nodes[t][i]["problem_global"] = np.asarray(npo[k])
            self.nodes[t][i]["global"] = np.asarray(npo[k])
        for t in self.submaps:
            for s in self.submaps[t]:
                s["optimized"] = s["global"].copy()
        self.since_last = 0

    def node_poses(self, t):
        return np.array([n["global"] for n in self.nodes.get(t, [])]).reshape(-1, 7)

    def submap_poses(self, t):
        """GetSubmapDataUnderLock: the optimized pose, else extrapolated with the trajectory's local-to-global transform."""
        l2g = self.local_to_global(t)
        return np.array([s["optimized"] if s["optimized"] is not None else compose(l2g, s["local"])
                         for s in self.submaps.get(t, [])]).reshape(-1, 7)
