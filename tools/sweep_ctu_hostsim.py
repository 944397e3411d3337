#!/usr/bin/env python
"""Randomised option sweep of the CTU search driver (host test build) against the unmodified reference encoder:
random picture sizes, QPs 8-48, smooth / noisy content, every preset, 0-4 random options inside the driver's scope
(rd level, PU depths, SAO / deblock / RDOQ / sign hiding / transform skip switches, full intra search, early terminations);
the two .hevc files must be equal.  CPU only (needs oracle/_ref built from /root/reference).

    python tools/sweep_ctu_hostsim.py <seed> <count> [--bitdepth 10]

--bitdepth 10: the 10-bit builds of the reference (kvazaar_10b / kvazaar_ctu_10b); the input is genuine 10-bit content
(--input-bitdepth 10) or, in a third of the runs, 8-bit content that the reference shifts up.

Round 2: seeds 1-13 and 20-39, 3000 configurations (plus QP 0-6 / 49-51 and extreme content: tools/sweep_ctu_content.py).  Seeds 5 and 8 found one bug (chroma mode search, --intra-chroma-search: scan order of the
candidates, fixed in csrc/ctu/ctu_search.h and covered by tests/test_ctu_driver.py::test_hostbuild_chroma_mode_search); 0 differences since.
"""
import sys, os, tempfile, pathlib, random
ROOT=os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0,os.path.join(ROOT,'tests')); sys.path.insert(0,os.path.join(ROOT,'tools'))
import test_ctu_driver as T
TEN='--bitdepth' in sys.argv and sys.argv[sys.argv.index('--bitdepth')+1]=='10'
if TEN:
    i=sys.argv.index('--bitdepth'); del sys.argv[i:i+2]
    import test_ctu_driver_10bit as T10
tmp=pathlib.Path(tempfile.mkdtemp(prefix='kvzs_', dir='/tmp'))
ref_bin, ctu_bin = [os.path.join(T.REF_DIR,n+('_10b' if TEN else '')) for n in ("kvazaar","kvazaar_ctu")]
rnd=random.Random(int(sys.argv[1]) if len(sys.argv)>1 else 1)
opts_pool=[["--rd","1"],["--rd","2"],["--rd","3"],["--rd","0"],["--pu-depth-intra","2-3"],["--pu-depth-intra","1-2"],["--pu-depth-intra","3-4"],["--no-sao"],["--sao","edge"],["--sao","band"],
 ["--no-deblock"],["--deblock","-2:1"],["--deblock","3:-3"],["--no-rdoq"],["--rdoq"],["--no-signhide"],["--signhide"],["--transform-skip"],["--no-transform-skip"],["--full-intra-search"],
 ["--intra-rdo-et"],["--cu-split-termination","off"],["--rdoq-skip"],["--no-rdoq-skip"],["--no-combine-intra-cus"],["--intra-chroma-search"],["--no-intra-chroma-search"]]
presets=["ultrafast","superfast","veryfast","faster","fast","medium","slow","slower","veryslow","placebo"]
n=int(sys.argv[2]) if len(sys.argv)>2 else 30
bad=0; inactive=0
for it in range(n):
    w=rnd.choice([64,72,128,136,200,264]); h=rnd.choice([64,72,128,136])
    qp=rnd.randint(8,48); noisy=rnd.random()<0.4; preset=rnd.choice(presets)
    extra=[]
    for o in rnd.sample(opts_pool, rnd.randint(0,4)): extra+=o
    frames=rnd.choice([1,1,2,3])
    extra+=['--threads',str(rnd.choice([0,1,2,4])),'--owf',str(rnd.choice([0,1,2,3]))]      # the hooks' picture slots and worker threads
    if TEN:
        ibd=rnd.choice([10,10,8])
        clip=T10._clip(tmp,w,h,frames,noisy,ibd)
        extra+=['--input-bitdepth',str(ibd)]
    else:
        clip=T._clip(tmp,w,h,frames,noisy)
    a,b=str(tmp/'a.hevc'),str(tmp/'b.hevc')
    try:
        T._encode(ref_bin,clip,w,h,a,preset,qp,extra=extra)
        log=T._encode(ctu_bin,clip,w,h,b,preset,qp,env={"KVZ_CTU_PROVIDER":(T10 if TEN else T)._hostsim()},extra=extra)
    except AssertionError as e:
        print('ENCODE FAIL',preset,w,h,qp,noisy,extra,str(e)[-300:],flush=True); bad+=1; continue
    active="CTU search driver active" in log
    same=open(a,'rb').read()==open(b,'rb').read()
    if not active: inactive+=1
    if not same:
        bad+=1
        print('DIFF',preset,w,h,qp,noisy,extra,'active',active,flush=True)
print('done',n,'bad',bad,'inactive',inactive,flush=True)
