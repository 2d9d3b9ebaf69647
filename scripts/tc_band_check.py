"""CPU check of the tensor-core graph filter's undecided band (DESIGN.md §3.1, prep_kernel): the FP32 evaluation of
d = t^2 - 2 beta^2 s + beta^4 and of band = kap (t^2 + beta^4) + c0 is emulated in numpy on squared norms perturbed by the
worst-case tensor-core error (+-e_a, +-e_b in every sign pattern and at random); a decided pair must agree with the exact
predicate.  usage: python scripts/tc_band_check.py"""
import numpy as np, sys, importlib
sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
synth=importlib.import_module("teaser-plusplus_b200.synth")
u=2.0**-24
KAPPA=64.0  # kTcKappa (csrc/tzr_internal.cuh)
def f32(x): return np.asarray(x,dtype=np.float64).astype(np.float32).astype(np.float64)
def check(src,dst,nb,mode,label,verbose=True):
    n=len(src); beta=2*nb
    mn=src.min(0);mx=src.max(0);Ds2=((mx-mn)**2).sum()
    mn=dst.min(0);mx=dst.max(0);Dd2=((mx-mn)**2).sum()
    E=KAPPA*u*(Ds2+Dd2); b2=beta*beta;b4=b2*b2
    lam=0.75*beta*np.sqrt(0.5*(Ds2+Dd2)); Smax=Ds2+Dd2+E
    kap=E/lam+8*u; c0=E*lam+E*E+2*b2*E+16*u*b2*Smax+8*u*b4+b4
    up=1+2.0**-20
    Dmin=np.sqrt(min(Ds2,Dd2))
    ok = 8*beta<=Dmin and 64*E<=0.75*Dmin*beta
    c2f=f32(2*b2); b4f=f32(b4); kapf=f32(kap*up); c0f=f32(c0*up)
    iu=np.triu_indices(n,1)
    a=((src[iu[0]]-src[iu[1]])**2).sum(1); b=((dst[iu[0]]-dst[iu[1]])**2).sum(1)
    exact=np.abs(np.sqrt(a)-np.sqrt(b))<=beta
    rng=np.random.default_rng(1)
    ea=KAPPA*u*Ds2; eb=KAPPA*u*Dd2
    if mode=='rand': pa=rng.uniform(-1,1,a.shape)*ea; pb=rng.uniform(-1,1,a.shape)*eb
    elif mode=='pp': pa=ea;pb=-eb
    elif mode=='pm': pa=-ea;pb=eb
    elif mode=='mm': pa=-ea;pb=-eb
    else: pa=ea;pb=eb
    ap=f32(a+pa); bp=f32(b+pb)
    t=f32(ap-bp); s=f32(ap+bp)
    P=f32(t*t+b4f); d=f32(P-c2f*s); bd=f32(P*kapf+c0f)
    dh=f32(d+bd); dl=f32(d-bd)
    sure_edge=np.signbit(dh); maybe=np.signbit(dl)
    sure_non=~maybe
    bad1=(sure_edge&~exact).sum(); bad2=(sure_non&exact).sum()
    und=(maybe&~sure_edge).sum()
    if verbose: print(f"{label:10s} {mode:4s} use_tc={ok} pairs={len(a)} edges={exact.sum()} undecided={und} ({und/len(a):.2e}) wrong_edge={bad1} wrong_non={bad2}")
    return int(bad1+bad2), float(und/len(a)), bool(ok)
def check_(*a):
    return check(*a)[0]

def main():
    tot=0
    for cfg,n in [("C2",1500),("C2cube",1100),("C3",2000),("C4",640),("C5",1700)]:
        pr=synth.config_problem(cfg,21,n=n)
        for mode in ['rand','pp','pm','mm','x']:
            tot+=check_(pr['src'],pr['dst'],pr['noise_bound'],mode,cfg)
    # duplicates / short TIMs
    pr=synth.config_problem("C2cube",8,n=700); src,dst=pr['src'].copy(),pr['dst'].copy()
    for k in range(0,60,3): src[k+1]=src[k]
    for k in range(100,160,3): dst[k+1]=dst[k]; src[k+1]=src[k]+1e-9
    for mode in ['rand','pp','pm']: tot+=check_(src,dst,pr['noise_bound'],mode,'dups')
    # big beta (beyond guard) to exercise s<=beta^2 clause
    pr=synth.config_problem("C2",3,n=600)
    for nb in [0.05,0.2,0.5]:
        for mode in ['rand','pm','pp']: tot+=check_(pr['src'],pr['dst'],nb,mode,f'nb{nb}')
    print('TOTAL WRONG',tot)

if __name__ == "__main__":
    main()
