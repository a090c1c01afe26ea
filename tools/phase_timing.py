import os, sys, numpy as np, torch
sys.path.insert(0, os.getcwd())
os.environ["VB200_PHASE_TIMING"]="1"
from vorbis_b200 import abi, lib
import bench
setup = abi.SetupHolder.load("tests/golden/setup_44k_stereo_q5.npz")
ctx = lib.Context(setup, 0)
N, ch, nb = 2048, 2, 20000
dev=torch.device("cuda",0)
pcm = bench.synth_pcm_torch(torch, nb, ch, N, 44100, dev, 1)
desc_np = bench.make_desc(nb)
desc = torch.from_numpy(desc_np.view(np.uint8).reshape(nb,16).copy()).to(dev)
outs=[torch.empty((nb,ch,N//2),device=dev) for _ in range(3)]; amp=torch.empty(nb,device=dev)
io=abi.PhaseAIO(); io.pcm,io.desc=pcm.data_ptr(),desc.data_ptr(); io.mdct,io.logmdct,io.logmask=(o.data_ptr() for o in outs); io.ampmax_out=amp.data_ptr()
for _ in range(3): ctx.phaseA_dev(1, nb, io)
ctx.debug_phase_cycles(True)
R=5
for _ in range(R): ctx.phaseA_dev(1, nb, io)
cyc = ctx.debug_phase_cycles(True)
rows = nb*ch*R
names=["load","runs","scatter","chase","grp_min","terms1","scan1","regress1","terms2","scan2","regress2+mix","  chase:records","  chase:simulate","  chase:fill"]
tot=sum(cyc[:11])
ghz=torch.cuda.get_device_properties(0).clock_rate/1e6  # the device's maximum SM clock: times are lower bounds
for n,c in zip(names,cyc): print("%-14s %8.0f cycles/row  %5.1f%%  (%.2f us @%.3fGHz)"%(n,c/rows,100*c/tot,c/rows/ghz/1e3,ghz))
print("total %.0f cycles/row = %.1f us"%(tot/rows, tot/rows/ghz/1e3))
