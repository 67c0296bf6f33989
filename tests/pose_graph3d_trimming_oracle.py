"""numpy restatement of mapping::PoseGraph3D's pure-localization bookkeeping, the counterpart of the dl_pg3d_* calls: the
bookkeeping of pose_graph3d_oracle.py over ids with holes (MapById, C/mapping/id.h:279-304), TrimmingHandle::
MarkSubmapAsTrimmed (pose_graph_3d.cc:1002-1058), PureLocalizationTrimmer (pose_graph_trimmer.cc:24-45) run after every
optimization (:492-501), FinishTrajectory (:535-547) and SetInitialTrajectoryPose with GetInterpolatedGlobalTrajectoryPose
(:849-876, :914-928). Submaps and nodes are dicts index -> record per trajectory; dict order is index order because indices
are only ever appended. The device stages are injected as in pose_graph3d_oracle.py."""
import numpy as np

from pose_graph3d_oracle import IDENTITY, INTER, INTRA, compose, inverse, pose_guess


class Rejected(Exception):
    """A call the device refuses with DL_ERR_ARG, the graph unchanged."""


def slerp(a, b, t):
    """Eigen's QuaternionBase::slerp (wxyz), in the dot order of the device helper (dl_pipeline.cuh)."""
    d = (a[1] * b[1] + a[2] * b[2]) + (a[3] * b[3] + a[0] * b[0])
    abs_d = abs(d)
    if abs_d >= 1.0 - 2.220446049250313e-16:
        s0, s1 = 1.0 - t, t
    else:
        theta = np.arccos(abs_d)
        st = np.sin(theta)
        s0, s1 = np.sin((1.0 - t) * theta) / st, np.sin(t * theta) / st
    if d < 0:
        s1 = -s1
    return np.array([s0 * a[0] + s1 * b[0], s0 * a[1] + s1 * b[1], s0 * a[2] + s1 * b[2], s0 * a[3] + s1 * b[3]])


def interpolate(times, poses, time):
    """GetInterpolatedGlobalTrajectoryPose: lower_bound by time, clamped at both ends, else transform::Interpolate."""
    k = next((i for i, t in enumerate(times) if not t < time), len(times))
    if k == 0:
        return np.array(poses[0], np.float64)
    if k == len(times):
        return np.array(poses[-1], np.float64)
    a, b = poses[k - 1], poses[k]
    f = (time - times[k - 1]) / (times[k] - times[k - 1])
    return np.concatenate([a[:3] + (b[:3] - a[:3]) * f, slerp(a[3:], b[3:], f)])


class PoseGraph3D:
    def __init__(self, optimize_every_n_nodes, every_nodes_to_find_constraint, matcher_weights=(5e2, 1.6e3)):
        self.n_opt, self.every = optimize_every_n_nodes, every_nodes_to_find_constraint
        self.weights = matcher_weights
        self.submaps = {}        # trajectory -> {index: dict(local, global, finished, node_ids, optimized)}
        self.nodes = {}          # trajectory -> {index: dict(time, local, global, problem_global)}
        self.next = {}           # trajectory -> [next submap index, next node index]
        self.can_append = {}     # trajectory -> [submaps, nodes]
        self.frozen = set()
        self.finished = set()
        self.initial = {}        # from trajectory -> (to trajectory, relative pose, time)
        self.trimmers = []       # [trajectory, num_submaps_to_keep], in the order added
        self.constraints = []    # (submap id, node id, zbar, tw, rw, tag)
        self.pending = []
        self.computed = {}
        self.since_last = 0
        self.searched = []
        self.solves = []
        self.last_trimmed = []

    # ---- SetInitialTrajectoryPose / ComputeLocalToGlobalTransform
    def set_initial_trajectory_pose(self, frm, to, relative, time):
        self.initial[frm] = (to, np.asarray(relative, np.float64), float(time))

    def local_to_global(self, t):
        for s in reversed(list(self.submaps.get(t, {}).values())):
            if s["optimized"] is not None:
                return compose(s["optimized"], inverse(s["local"]))
        if t not in self.initial:
            return IDENTITY.copy()
        to, rel, time = self.initial[t]
        nodes = list(self.nodes.get(to, {}).values())
        if not nodes:
            raise Rejected("the initial pose refers to a trajectory without nodes")
        return compose(interpolate([n["time"] for n in nodes], [n["global"] for n in nodes], time), rel)

    # ---- AddNode + ComputeConstraintsForNode
    def add_node(self, t, local_pose, insertion, matches=(), search=None, solve=None, time=0.0):
        local_pose = np.asarray(local_pose, np.float64)
        self.last_trimmed = []          # every call that may trim empties the list when it starts
        subs = self.submaps.get(t, {})
        nxt = self.next.get(t, [0, 0])
        app = self.can_append.get(t, [True, True])
        S = nxt[0]
        idx = [i for i, _, _ in insertion]
        if t in self.finished or not app[1]:
            raise Rejected("finished trajectory or node appends forbidden")
        if len(insertion) == 1:
            if idx != [0] or S > 1:
                raise Rejected("sequence")
            back_new = S == 0
        else:
            if not ((S >= 1 and idx == [S - 1, S]) or (S >= 2 and idx == [S - 2, S - 1])):
                raise Rejected("sequence")
            back_new = idx[1] == S
        if back_new and not app[0]:
            raise Rejected("submap appends forbidden")
        for i in idx:
            if i < S and (i not in subs or subs[i]["finished"]):
                raise Rejected("insertion submap trimmed or finished")
        for mt in matches:
            if mt[1] not in self.submaps.get(mt[0], {}) or not self.submaps[mt[0]][mt[1]]["finished"]:
                raise Rejected("a match names an unknown, trimmed or unfinished submap")
        l2g = self.local_to_global(t)
        # ---- commit
        subs = self.submaps.setdefault(t, {})
        nodes = self.nodes.setdefault(t, {})
        self.next[t], self.can_append[t] = nxt, app
        node_index = nxt[1]
        nxt[1] += 1
        node = {"time": float(time), "local": local_pose, "global": compose(l2g, local_pose)}
        if back_new:
            local = np.asarray(insertion[-1][2], np.float64)
            if len(insertion) == 1:
                g = compose(l2g, local)
            else:
                f = subs[idx[0]]
                g = compose(compose(f["global"], inverse(f["local"])), local)
            subs[S] = {"local": local, "global": g, "finished": False, "node_ids": [], "optimized": None}
            nxt[0] += 1
        m = subs[idx[0]]
        node["problem_global"] = compose(compose(m["global"], inverse(m["local"])), local_pose)
        nodes[node_index] = node
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
                live = [n for n in frm["node_ids"] if n in nodes]      # trimmed nodes are holes
                for j, n in enumerate(live):
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

    # ---- HandleWorkQueue + RunOptimization + trimmers
    def optimize(self, solve):
        for c in self.pending:
            if not any(c[0] == d[0] and c[1] == d[1] for d in self.constraints):
                self.constraints.append(c)
        self.pending = []
        sids = [(t, i) for t in sorted(self.submaps) for i in self.submaps[t]]
        nids = [(t, i) for t in sorted(self.nodes) for i in self.nodes[t]]
        if sids:
            sp = np.array([self.submaps[t][i]["global"] for t, i in sids])
            npo = np.array([self.nodes[t][i]["problem_global"] for t, i in nids]).reshape(-1, 7)
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
                for s in self.submaps[t].values():
                    s["optimized"] = s["global"].copy()
            self.since_last = 0
        self.run_trimmers()

    def run_trimmers(self):
        for tr in self.trimmers:
            if tr[0] in self.finished:
                tr[1] = 0
            ids = list(self.submaps.get(tr[0], {}))
            for i in range(len(ids)):
                if i + tr[1] < len(ids):
                    self.check_trimmable(tr[0], ids[i])
                    self.mark_submap_as_trimmed((tr[0], ids[i]))
        self.trimmers = [tr for tr in self.trimmers if tr[1] != 0]

    def add_pure_localization_trimmer(self, t, keep):
        if keep < 3:
            raise Rejected("keep >= 3")
        self.trimmers.append([t, keep])

    def finish_trajectory(self, t, solve):
        self.last_trimmed = []
        if t in self.finished:
            raise Rejected("finished twice")
        self.finished.add(t)
        for s in self.submaps.get(t, {}).values():
            s["finished"] = True
        self.optimize(solve)

    def run_final_optimization(self, solve):
        self.last_trimmed = []
        self.optimize(solve)

    # ---- MarkSubmapAsTrimmed
    def check_trimmable(self, t, i):
        if i not in self.submaps.get(t, {}):
            raise Rejected("unknown or trimmed submap")
        if not self.submaps[t][i]["finished"]:
            raise Rejected("unfinished submap")
        if self.pending:
            raise Rejected("constraints pending")

    def trim_submap(self, t, i):
        self.last_trimmed = []
        self.check_trimmable(t, i)
        self.mark_submap_as_trimmed((t, i))

    def mark_submap_as_trimmed(self, sid):
        retain = {c[1] for c in self.constraints if c[5] == INTRA and c[0] != sid}
        remove = {c[1] for c in self.constraints if c[0] == sid and c[5] == INTRA and c[1] not in retain}
        self.constraints = [c for c in self.constraints if c[0] != sid and c[1] not in remove]
        subs = self.submaps[sid[0]]
        if sid[1] == max(subs):
            self.can_append[sid[0]][0] = False
        del subs[sid[1]]
        self.computed.pop(sid, None)
        for nid in sorted(remove):
            nodes = self.nodes[nid[0]]
            if nid[1] == max(nodes):
                self.can_append[nid[0]][1] = False
            del nodes[nid[1]]
            for v in self.computed.values():
                v.discard(nid)
        self.last_trimmed.append(sid)

    # ---- queries
    def ids(self, t, nodes=True):
        return list((self.nodes if nodes else self.submaps).get(t, {}))

    def node_poses(self, t):
        return np.array([n["global"] for n in self.nodes.get(t, {}).values()]).reshape(-1, 7)

    def submap_poses(self, t):
        subs = list(self.submaps.get(t, {}).values())
        l2g = self.local_to_global(t) if subs else IDENTITY
        return np.array([s["optimized"] if s["optimized"] is not None else compose(l2g, s["local"]) for s in subs]).reshape(-1, 7)
