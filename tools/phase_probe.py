"""Per-phase cycle shares of the step kernel (needs a -DHWY_PHASE_TIMING build, see hwy_highway.cu):
  nvcc ... -DHWY_PHASE_TIMING -o highwayenv_b200/csrc/variants/lib_timing.so ...; HWYB200_LIB=that python tools/phase_probe.py"""
import ctypes as C, os, sys
sys.path.insert(0, os.getcwd())
import torch
import highwayenv_b200 as hb
from highwayenv_b200 import _native as N
env = hb.make("highway-fast-v0", num_envs=4096, config={"vehicles_count": 50})
env.reset(seed=0)
lib = env._lib
lib.hwy_debug_phase_cycles.argtypes=[C.c_void_p]
lib.hwy_debug_order_probe.argtypes=[C.c_void_p]
buf = (C.c_ulonglong*16)()
order = (C.c_ulonglong*4)()
g = torch.Generator(device="cuda"); g.manual_seed(1)
acts = torch.randint(0,5,(40,4096),generator=g,device="cuda",dtype=torch.int32)
for t in range(10): env.step(acts[t])
torch.cuda.synchronize(); lib.hwy_debug_phase_cycles(buf); lib.hwy_debug_order_probe(order)
for t in range(10,40): env.step(acts[t])
torch.cuda.synchronize(); lib.hwy_debug_phase_cycles(buf); lib.hwy_debug_order_probe(order)
names = ["load+static","publish","bar(publish)","build(rank/masks/sweep1)","bar(build)","sweep2","ego action","phase A1","bar(A1)","phase B","integrate","(loop exit)","epilogue","phase A2 (MOBIL items)","bar(A2)"]
tot = sum(buf)
for k,n in enumerate(names): print(f"{n:28s} {buf[k]/tot*100:5.1f}%")
print("cycles per warp per step:", tot/(30*4096*2))
frames, fails, counted, cyc = order
print(f"order: {frames} env-frames, chain check failed in {fails} ({fails/max(frames,1)*100:.1f} %), "
      f"rank_count in {counted} envs, {cyc} warp cycles recovering a failed order ({cyc/tot*100:.2f} % of the phases)")
