"""TEST INFRASTRUCTURE (not collected by pytest): randomised differential run of the scaler's whole-frame host call -- libav_b200/csrc/swscale.cu compiled
for the host (tests/hostsim/, built by tests/hostsim_build.py) -- against the compiled reference (oracle/_ref).  Random
source / destination format, geometry and flags; every request the product accepts must give the reference's picture bytes.
usage: python tests/fuzz_sws_hostsim.py [seed [requests]]        (round 2: seeds 1-12 and 21-23, ~18000 requests, ~14000 accepted; two findings, both fixed: slices into a gray8 destination, bgr24 -> gray8 at the same size)"""
import sys, os
HERE = os.path.dirname(os.path.abspath(__file__)); sys.path.insert(0, HERE); sys.path.insert(0, os.path.dirname(HERE))
import numpy as np, ctypes as C, random
from oracle import loader
import hostsim_build
import test_hostsim_sws_frames_cpu as H
import test_sws_plan_cpu as P
import test_sws_gray_src as G
import test_sws_pal8_src as PAL
from libav_b200 import synth
refo = loader.ref()
lib = hostsim_build.load()
SRCS = [0,4,5,6,7,31,12,13,14,32,33,8,11,23,24,1,15,2,3,25,26,27,28,62,61,64,63,47,48,66,70,72,68,49,51]
DSTS = [0,4,5,6,7,31,12,13,14,32,2,3,25,26,27,28,1,15,23,24,8,37,36,41,43,54,57,35,34,60,59,62,64,66,68,61,63,72,70]
SUB = {0:(1,1),4:(1,0),5:(0,0),6:(2,2),7:(2,0),31:(0,1),12:(1,1),13:(1,0),14:(0,0),32:(0,1),33:(1,1)}
def source(sf,w,h,seed):
    r=np.random.RandomState(seed)
    if sf>40:
        import test_sws_hbd_sources_cpu as HB
        return HB.planes(sf,w,h,seed)
    if sf==8: return [G.picture(w,h,seed)]
    if sf==11:
        i,p=PAL.picture(w,h,seed); return [i,p.view(np.uint8).reshape(1,1024)]
    if sf in (23,24):
        cw,ch=(w+1)//2,(h+1)//2
        return [synth.pad_rows(r.randint(0,256,(h,w)).astype(np.uint8)), synth.pad_rows(r.randint(0,256,(ch,2*cw)).astype(np.uint8))]
    if sf in (1,15): return [r.randint(0,256,(h,2*w+12)).astype(np.uint8)]
    if sf in (2,3): return [r.randint(0,256,(h,3*w+12)).astype(np.uint8)]
    if 25<=sf<=28: return [r.randint(0,256,(h,4*w+12)).astype(np.uint8)]
    hs,vs=SUB[sf]; cw,ch=-((-w)>>hs),-((-h)>>vs)
    return [synth.pad_rows(r.randint(0,256,s).astype(np.uint8)) for s in ((h,w),(ch,cw),(ch,cw))]
def outputs(df,dw,dh):
    if df in (12,13,14,32):
        hs,vs={12:(1,1),13:(1,0),14:(0,0),32:(0,1)}[df]; cw,ch=-((-dw)>>hs),-((-dh)>>vs)
        return [np.full((dh,dw+8),7,np.uint8),np.full((ch,cw+8),7,np.uint8),np.full((ch,cw+8),7,np.uint8)]
    if df==8: return [np.full((dh,dw+16),7,np.uint8)]
    return H.outputs(df,dw,dh,pad=8) if 'pad' in H.outputs.__code__.co_varnames else H.outputs(df,dw,dh)
rnd=random.Random(int(sys.argv[1]) if len(sys.argv)>1 else 1)
N=int(sys.argv[2]) if len(sys.argv)>2 else 400
acc=bad=0
for it in range(N):
    sf=rnd.choice(SRCS); df=rnd.choice(DSTS)
    w=rnd.choice([16,17,34,64,65,100,131]); h=rnd.choice([8,9,16,33,48,50])
    if rnd.random()<0.35: dw,dh=w,h
    else: dw=rnd.choice([16,24,33,64,96,130,200]); dh=rnd.choice([8,12,25,48,64,97])
    flags=rnd.choice([1,2,4,0x10,0x20,0x40,0x200,0x400])|rnd.choice([0,0x40000,0x80000,0xC0000])|rnd.choice([0,0,0x2000])|rnd.choice([0,0,0,0x4000])
    if flags&1 and (sf in (23,24,1,15,2,3,25,26,27,28,11)) and dw>w: continue
    if flags&1 and sf in (1,15,2,3,25,26,27,28,23,24,11): 
        # chroma upscale may also hit the undefined edge
        continue
    ctx=lib.sws_getContext_cuda(w,h,sf,dw,dh,df,flags,None,None,None)
    if not ctx:
        lib.avb200_clear_error() if hasattr(lib,'avb200_clear_error') else None
        continue
    pl=source(sf,w,h,it)
    got=outputs(df,dw,dh); want=outputs(df,dw,dh)
    flip = rnd.random() < 0.25 and sf != 11          # bottom-up pictures (negative strides) on both sides
    if flip:
        store = [np.ascontiguousarray(o[::-1]) for o in got]
        gv = [g[::-1] for g in store]
        sv = [np.ascontiguousarray(a[::-1])[::-1] for a in pl]
        sp,ss=H.arrays(sv); dp,ds=H.arrays(gv)
    else:
        sp,ss=H.arrays(pl); dp,ds=H.arrays(got)
    r=lib.sws_scale_cuda(ctx,sp,ss,0,h,dp,ds)
    if flip: got = [np.ascontiguousarray(g) for g in gv]
    lib.sws_freeContext_cuda(ctx)
    sp3=(C.c_void_p*3)(*([a.ctypes.data for a in pl]+[None]*(3-len(pl)))); ss3=(C.c_int*3)(*([a.strides[0] for a in pl]+[0]*(3-len(pl))))
    dp3=(C.c_void_p*3)(*([a.ctypes.data for a in want]+[None]*(3-len(want)))); ds3=(C.c_int*3)(*([a.strides[0] for a in want]+[0]*(3-len(want))))
    rr=refo.sws_planar(sf,sp3,ss3,w,h,df,dp3,ds3,dw,dh,flags)
    acc+=1
    ok = r==dh==rr
    if ok:
        bpp = 6 if df in (34,35,59,60) else 4 if 25<=df<=28 else 2 if df in (1,15) or 36<=df<=43 or 54<=df<=57 else 3 if df in (2,3) else 0
        for a,b in zip(got,want):
            cut = bpp*dw if bpp and len(got)==1 else a.shape[1]-8          # the picture, not the row padding (the reference's one-call converters also convert that)
            a2,b2=a[:, :cut], b[:, :cut]
            if not np.array_equal(a2,b2): ok=False; where=np.argwhere(a2!=b2)[:3].tolist(); break
    if not ok:
        bad+=1
        print("DIFF", sf, df, w,h,dw,dh,hex(flags), r, rr, locals().get('where'))
print("accepted", acc, "bad", bad)
