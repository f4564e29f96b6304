"""Seeded drives for the window upkeep (tests/test_track_upkeep.py, scripts/upkeep_bench.py): deactivateKeyframes and the AddDepth
scheme with ground labels.

An UpkeepDrive is a tests/create_drive.Drive (its landmarks cover push()'s creation cases, NaN positions among them) with:
  - long-lived landmarks, 8 per push, seen by camera 0 for 25 keyframes: they keep every keyframe connected to the newest one up
    to max_window, so that the window rule is what deactivates most keyframes;
  - a gap keyframe that measures none of them: once six keyframes newer, it shares no landmark with the newest one and the
    connection rule (common <= min_connecting) deactivates it inside the window;
  - a bare keyframe whose landmarks are not ground: it has no eligible landmark;
  - tie pairs: a copy, under a new id, of a landmark with a depth on every camera, measured identically -- both are created at
    the same position, so their costs tie;
  - ground labels: every landmark except those of the bare keyframe, the long-lived ones and the untied ids = 1 mod 3.
write() adds one line `ground N id ...` to the file format of create_drive.Drive (tests/cpp/test_facade_upkeep.cpp reads it)."""
import numpy as np

from tests.create_drive import F32, Drive, _rot


class UpkeepDrive(Drive):
    def __init__(self, seed, n_push=30, window=12, rig=True, new_per_push=40):
        super().__init__(seed, n_push=n_push, window=window, rig=rig, new_per_push=new_per_push)
        rng = np.random.default_rng(seed + 1000)
        self.gap, self.bare = n_push // 3, n_push // 3 + 2
        lm = self.n_lm
        long_lived, ties = set(), []
        for k in range(n_push):
            for _ in range(8):
                p = np.array([1.5 * k + rng.uniform(60, 100), rng.uniform(-10, 10), rng.uniform(-2, 5)])
                for kk in range(k, min(n_push, k + 25)):
                    if kk == self.gap:
                        continue
                    Rk, tk = _rot(self.kf_pose[kk][:4]), self.kf_pose[kk][4:]
                    Rc, tc = _rot(self.cam_pose[0][:4] / np.linalg.norm(self.cam_pose[0][:4])), self.cam_pose[0][4:]
                    pc = Rc @ (Rk @ p + tk) + tc
                    f, cx, cy = self.cam_intr[0]
                    u, v = f * pc[0] / pc[2] + cx + rng.normal(0, 0.5), f * pc[1] / pc[2] + cy + rng.normal(0, 0.5)
                    self.meas[kk][lm] = [(0, F32(u), F32(v), F32(-1.0))]
                long_lived.add(lm)
                lm += 1
            # a landmark first seen here with a depth on every camera, copied under a new id
            first = [lid for lid, obs in self.meas[k].items() if lid < self.n_lm and all(o[3] >= 0 for o in obs)]
            if first:
                src = first[0]
                for kk in range(k, n_push):
                    if src in self.meas[kk]:
                        self.meas[kk][lm] = list(self.meas[kk][src])
                ties.append((src, lm))
                lm += 1
        self.n_lm, self.ties = lm, ties
        tied = {x for pair in ties for x in pair}
        bare = set(self.meas[self.bare])
        self.ground = np.array([lid not in bare and (lid in tied or (lid not in long_lived and lid % 3 != 1)) for lid in range(lm)])

    def write(self, path):
        super().write(path)
        ids = np.flatnonzero(self.ground)
        with open(path, "a") as f:
            f.write("ground %d %s\n" % (len(ids), " ".join(str(i) for i in ids)))
