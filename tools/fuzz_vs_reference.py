#!/usr/bin/env python3
"""Randomised cross-check of the host logic and the CPU oracle against the UNMODIFIED reference (oracle/_ref, so only
where /root/reference was available at build time): random cjpeg switch sets on random small images through
(a) the reference's own cjpeg binary and (b) the cjpeg mirror + b200jpeg_validate + the oracle; a quarter of the cases use the CMYK / YCCK / YCbCr->gray /
JCS_UNKNOWN conversions (reference: build/librefcs.so, the switches tests/refcs.c knows).  Test infrastructure.
usage: fuzz_vs_reference.py [seed] [cases]      (exit status 1 if anything differs)"""
import os, random, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
from oracle import oracle as O
import mozjpeg_b200 as mj
from mozjpeg_b200 import _abi as A
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import colorspace_cases as CC       # the other colour conversions: reference through build/librefcs.so
rng=random.Random(int(sys.argv[1]) if len(sys.argv)>1 else 1)
lib=A.load()
bad=0; tot=0; refused=0
for it in range(int(sys.argv[2]) if len(sys.argv)>2 else 150):
    w=rng.choice([1,7,8,16,17,33,64,100,131]); h=rng.choice([1,5,8,16,23,40,64,77])
    im=O.synth_image(rng.randrange(1<<20),w,h)
    sw=[]
    prof=rng.choice(["", "-revert", "-baseline", "-fastcrush", "-progressive"])
    if prof=="-progressive": sw+=["-revert","-progressive"] if rng.random()<0.5 else ["-progressive"]
    elif prof: sw.append(prof)
    if rng.random()<0.8: sw+=["-quality",str(rng.choice([5,20,40,60,75,80,85,90,95,100]))]
    if rng.random()<0.5: sw+=["-sample",rng.choice(["1x1","2x1","1x2","2x2","3x1","4x2","2x2,1x1,2x2","1x1,2x1,1x1","4x1,2x1,1x1"])]
    if rng.random()<0.2: sw+=["-grayscale"]
    if rng.random()<0.25: sw+=["-restart",rng.choice(["1","2","3B","7B","1B"])]
    if rng.random()<0.2: sw+=["-dct",rng.choice(["fast","float","int"])]
    if rng.random()<0.15: sw+=["-smooth",str(rng.choice([1,10,50,100]))]
    if rng.random()<0.15: sw+=[rng.choice(["-notrellis","-notrellis-dc","-noovershoot","-optimize","-nojfif","-quant-baseline"])]
    if rng.random()<0.1: sw+=["-quant-table",str(rng.randrange(0,9))]
    if rng.random()<0.1: sw+=[rng.choice(["-tune-psnr","-tune-ssim","-tune-ms-ssim","-tune-hvs-psnr"])]
    if rng.random()<0.1: sw+=["-dc-scan-opt",str(rng.randrange(0,3))]
    if rng.random()<0.1: sw+=["-trellis-dc-ver-weight",rng.choice(["0.5","1.0","3"])]
    if rng.random()<0.1: sw+=["-lambda1",rng.choice(["9","12.5","14.75"]),"-lambda2",rng.choice(["0","13","16.5"])]
    conv=rng.choice(list(CC.CONVERSIONS)) if CC.have_reference() and rng.random()<0.25 else None
    if conv:
        sw=[x for x in sw if x not in ("-grayscale","-nojfif","-quant-baseline") and not x.startswith("-tune") and x!="-notrellis-dc"]
        sw=[x for i,x in enumerate(sw) if not (x.startswith("-") and x[1:] in ("quant-table","dc-scan-opt","trellis-dc-ver-weight","lambda1","lambda2")) and not (i>0 and sw[i-1][1:] in ("quant-table","dc-scan-opt","trellis-dc-ver-weight","lambda1","lambda2"))]
        in_cs,ic,jcs=CC.CONVERSIONS[conv]; im=CC.cmyk_image(rng.randrange(1<<20),w,h,ic)
    try:
        a=CC.ref_encode(im,in_cs,ic,jcs,sw) if conv else O._ref_cjpeg_pixels(im,sw); ref_ok=True
    except Exception as ex:
        a=None; ref_ok=False; referr=str(ex).strip().splitlines()[-1][-70:]
    try:
        p=mj.params_from_switches(sw,w,h,ic,in_cs,jcs) if conv else mj.params_from_switches(sw,w,h,3)
    except Exception as ex:
        if ref_ok: print("MIRROR REJECTS what reference accepts:",sw,ex); bad+=1
        continue
    rc=lib.b200jpeg_validate(C.byref(p))
    if not ref_ok:
        if rc==0: print("WE ACCEPT what reference rejects:",sw,(w,h),referr); bad+=1
        continue
    if rc!=0:
        refused+=1
        if rc==-1: print("WE REJECT (PARAM) what reference accepts:",sw,(w,h),lib.b200jpeg_last_error()); bad+=1
        continue
    tot+=1
    try: b=CC.oracle_encode(p,im).jpeg
    except Exception as ex: print("ORACLE FAIL",sw,(w,h),ex); bad+=1; continue
    if a!=b: bad+=1; print("MISMATCH",sw,(w,h),len(a),len(b))
print("seed", sys.argv[1:], "bad", bad, "compared", tot, "refused(unsupported)", refused)
sys.exit(1 if bad else 0)
