"""precision = 1 (FP32 residual / Jacobian blocks, FP64 accumulation) against the FP64 solve and the oracle"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from limo_b200 import synth, capi
h = capi.Handle(0)
o32 = capi.default_options(); o32.precision = 1
for name, win in (("config2", synth.make_window(2)), ("config3", synth.make_window(3, seed=41)), ("config1", synth.make_window(1))):
    r64 = h.solve_window(win); r32 = h.solve_window(win, o32)
    dt = np.linalg.norm(r32.kf_pose[:, 4:] - r64.kf_pose[:, 4:], axis=1).max()
    dl = np.linalg.norm(r32.lm_pos[:win.n_lm] - r64.lm_pos[:win.n_lm], axis=1)
    print(name, "iters 64/32", [s.num_iterations for s in r64.solves], [s.num_iterations for s in r32.solves],
          "final cost rel diff %.3e" % (abs(r32.c.final_cost - r64.c.final_cost) / r64.c.final_cost),
          "max dt %.3e" % dt, "p95 dlm %.3e" % np.percentile(dl, 95),
          "rejected differ %d of %d" % (int((r32.lm_rejected != r64.lm_rejected).sum()), win.n_lm),
          "device ms 64/32 %.2f %.2f" % (1e3 * r64.c.time_sec, 1e3 * r32.c.time_sec))
win = synth.make_window(2, n_kf=12, n_lm=400, n_obs=3000)
a = h.evaluate(win); b = h.evaluate(win, o32)
print("eval: cost rel %.2e  |dr| %.2e  |djp|/max %.2e  |djl|/max %.2e" % (abs(a[3] - b[3]) / a[3], np.abs(a[0] - b[0]).max(),
      np.abs(a[1] - b[1]).max() / np.abs(a[1]).max(), np.abs(a[2] - b[2]).max() / np.abs(a[2]).max()))
wins = [synth.make_window(2, seed=0xBA5E0000 + i) for i in range(16)]
batch = h.batch([wins[i % 16] for i in range(132)])
for opt, nm in ((capi.default_options(), "fp64"), (o32, "fp32-lin")):
    for _ in range(2): batch.solve(opt)
    t = time.time(); batch.solve(opt); batch.solve(opt); dtm = (time.time() - t) / 2
    print(nm, "132-window batch: %.1f ms per solve -> %.0f windows/s" % (1e3 * dtm, 132 / dtm))
batch.close(); h.close()
