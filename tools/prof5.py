import sys, ctypes
sys.path.insert(0,'.')
from pop_up_slam_b200 import graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI
# usage: prof5.py [timer_cta]  -- the CTA whose thread 0 keeps the timers (the look-ahead slot is non-zero only on CTAs that
# own a diagonal tile of A_c)
rank = int(sys.argv[1]) if len(sys.argv) > 1 else 0
g = gg.make_config(3, seed=0)
a = GpuGraphAPI(); gg.build_bulk(a, g); gg.configure(a, g)
o = a.get_solver_options(); o.reserved[2] = 1 | (rank << 8)
a._chk(a.lib.pus_set_solver_options(a.h, ctypes.byref(o)))
a.upload(); a.debug_run_stage(1, 1e-6)
st = a.stats(); ph = st['phase_ms']
steps = int(a.debug_fetch("dims", 14)[13]) * 6 // 48
print("one setup: Hinv %.3f blocks %.3f Wc %.3f Ac %.3f AcInv %.3f ms"%(ph[8],ph[9],ph[10],ph[11],ph[12]))
print(" AcInv parts on CTA %d (%d steps): P + T rows %.1f  diagonal update + pivot inverse %.1f  tile update + snapshot %.1f  barrier %.1f us/step"
      % ((rank, steps) + tuple(ph[k]*1e3/steps for k in (7,6,21,22))))
