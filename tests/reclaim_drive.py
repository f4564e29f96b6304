"""Long drives for the landmark slot reclaim (tests/test_track_reclaim.py, scripts/reclaim_bench.py).

A ReclaimDrive is a tests/create_drive.Drive (its landmarks cover push()'s creation cases) with revisited landmarks: 4 per push,
far ahead, seen by camera 0 in three consecutive keyframes and again in two keyframes more than a ring of keyframe slots later,
so that every keyframe of the first visit has left the store before the second (some with a lidar depth on the first visit).

SlotBook is a caller that keeps no host copy of the measurements and has fewer landmark slots than the drive has landmarks: it
hands slots out densely, then from a LIFO free list (so slot order is not id order), and when a push needs more slots than it
has, asks `reclaim(lo, hi)` for the free ones of [0, slots handed out) and evicts their landmarks.  `reclaim` is the device
(Track.reclaim_landmarks) or free_slots() below, the statement of what the device returns."""
import numpy as np

from tests.create_drive import F32, Drive, _rot


def free_slots(live_arenas, lo, hi):
    """the slots in [lo, hi) that no arena entry of a live keyframe names, ascending"""
    named = set()
    for lm in live_arenas:
        named.update(int(s) for s in lm)
    return np.array([s for s in range(lo, hi) if s not in named], np.int32)


class ReclaimDrive(Drive):
    def __init__(self, seed, n_push=90, window=8, rig=True, new_per_push=40):
        super().__init__(seed, n_push=n_push, window=window, rig=rig, new_per_push=new_per_push)
        rng = np.random.default_rng(seed + 2000)
        ring = window + 2
        lm = self.n_lm
        self.revisited = set()
        for k in range(n_push):
            for j in range(4):
                p = np.array([1.5 * k + rng.uniform(70, 110), rng.uniform(-10, 10), rng.uniform(-2, 4)])
                back = k + 2 + ring + 2 + (j + k) % 4
                visits = [kk for kk in [k, k + 1, k + 2, back, back + 1] if kk < n_push]
                for i, kk in enumerate(visits):
                    Rk, tk = _rot(self.kf_pose[kk][:4]), self.kf_pose[kk][4:]
                    Rc, tc = _rot(self.cam_pose[0][:4] / np.linalg.norm(self.cam_pose[0][:4])), self.cam_pose[0][4:]
                    pc = Rc @ (Rk @ p + tk) + tc
                    f, cx, cy = self.cam_intr[0]
                    u, v = f * pc[0] / pc[2] + cx + rng.normal(0, 0.5), f * pc[1] / pc[2] + cy + rng.normal(0, 0.5)
                    d = pc[2] + rng.normal(0, 0.05) if (i == 0 and j % 2 == 0) else -1.0
                    self.meas[kk][lm] = [(0, F32(u), F32(v), F32(d))]
                if back < n_push:
                    self.revisited.add(lm)
                lm += 1
        self.n_lm = lm


class SlotBook:
    """landmark id -> slot of a caller with `cap` landmark slots (see the module docstring)"""

    def __init__(self, cap):
        self.cap = cap
        self.slot = {}                    # landmark id -> slot
        self.owner = []                   # slot -> the landmark id it was handed to last
        self.free = []                    # LIFO
        self.evicted = {}                 # landmark id -> (pos, weight) kept at its eviction
        self.reclaims = 0
        self.restored = set()             # ids that got a slot again after an eviction

    def assign(self, ids, reclaim):
        """slots for `ids` (one keyframe's landmarks, ascending); reclaim(lo, hi) -> (slots, pos, weight) of the free slots.
        Returns (slots of ids, [(id, slot, pos, weight)] of evicted landmarks that got a slot again)."""
        need = [i for i in ids if i not in self.slot]
        if len(need) > len(self.free) + self.cap - len(self.owner):
            slots, pos, weight = reclaim(0, len(self.owner))
            self.reclaims += 1
            keep = set(ids)
            for s, p, w in zip(slots, pos, weight):
                lid = self.owner[s]
                if self.slot.get(lid) != s or lid in keep:   # free already, or measured by the keyframe being pushed
                    continue
                del self.slot[lid]
                self.evicted[lid] = (np.array(p), float(w))
                self.free.append(int(s))
            if len(need) > len(self.free) + self.cap - len(self.owner):
                raise RuntimeError("SlotBook: %d landmark slots cannot hold one keyframe's new landmarks" % self.cap)
        back = []
        for lid in need:
            if self.free:
                s = self.free.pop()
                self.owner[s] = lid
            else:
                s = len(self.owner)
                self.owner.append(lid)
            self.slot[lid] = s
            if lid in self.evicted:
                p, w = self.evicted.pop(lid)
                back.append((lid, s, p, w))
                self.restored.add(lid)
        return np.array([self.slot[i] for i in ids], np.int32), back
