"""Python emulation of the radix-2^32 lane-distributed Montgomery product of
bftkv_b200/csrc/mont_r32.cuh (same E/O/Z/cin bookkeeping), checked against big-int arithmetic.
`owners` < T stops after that many owner steps, as K1's final check does; mont_finish_emu merges the accumulators and
resolves the carries across the lanes limb for limb (mont_finish), group_sub_emu / cond_sub_emu are group_sub / cond_sub.

W (32-bit limbs per lane) is 16 for 2048-bit numbers (K1, K5 at 2048 bits) and 8 for 1024-bit ones (K5 at 1024 bits,
both CRT halves of K6a).  The lane-level helpers take it from their operands; the product and `lanes` take it as an
argument.

`trace`: an optional collections.Counter.  mont_finish_emu, group_sub_emu, group_ge_emu and cond_sub_emu add one count
per (event, lane) they take, so a caller can tell which carry and borrow paths an operand reached:
    finish_carry_gen    the lane's merge generated a carry into the lane above (lane T - 1: into bit 128 W)
    finish_carry_prop   an all-ones lane passed the carry that came in on to the lane above (p[r] and ci[r])
    finish_overflow     the result reached 2^(128 W) and n was subtracted (lane None)
    finish_borrow_gen   during that subtraction, a lane generated a borrow
    finish_borrow_prop  during that subtraction, a borrow passed through a lane of zeros
    sub_borrow_gen / sub_borrow_prop        the same for group_sub_emu called directly (cond_sub: cond_borrow_*)
    cond_sub_taken / cond_sub_skipped       cond_sub_emu did or did not subtract n (lane None)
    ge_below_top        group_ge was decided by a lane below the top one (the deciding lane)
    ge_equal            group_ge found all lanes equal (lane None)"""
import random
B=1<<32; T=4; W=16
def chain(arr, idxpairs, xs, m, c=0):
    for lo,xi in idxpairs:
        v = arr[lo] + (arr[lo+1]<<32) + xs[xi]*m + c
        arr[lo]=v&(B-1); arr[lo+1]=(v>>32)&(B-1); c=v>>64
    return c
def end(arr, idx, c, n2):
    for k in range(n2):
        v=arr[idx+k]+c; arr[idx+k]=v&(B-1); c=v>>32
    assert c==0
def montmul_acc(a,b,n,n0inv, owners=T, W=W):
    """the accumulators (E, O, Z, cin) after `owners` owner steps"""
    al=lanes(a,W); bl=lanes(b,W); nl=lanes(n,W)
    E=[[0]*(W+3) for _ in range(T)]; O=[[0]*(W+1) for _ in range(T)]; cin=[0]*T; Z=[0]*T
    rnd=0
    for owner in range(owners):
        for jj in range(0,W,2):
            b0=bl[owner][jj]; b1=bl[owner][jj+1]
            for r in range(T):
                c=chain(E[r], [(k,k) for k in range(0,W,2)], al[r], b0, cin[r]); end(E[r],W,c,2)
            q0=(((E[0][0]+Z[0])&(B-1))*n0inv)&(B-1)
            for r in range(T):
                c=chain(O[r], [(k-1,k) for k in range(1,W,2)], al[r], b0); end(O[r],W,c,1)
                c=chain(O[r], [(k,k) for k in range(0,W,2)], al[r], b1); end(O[r],W,c,1)
                c=chain(E[r], [(k+1,k) for k in range(1,W,2)], al[r], b1); end(E[r],W+2,c,1)
                c=chain(E[r], [(k,k) for k in range(0,W,2)], nl[r], q0); end(E[r],W,c,2)
                c=chain(O[r], [(k-1,k) for k in range(1,W,2)], nl[r], q0); end(O[r],W,c,1)
            s0=[E[r][0]+Z[r] for r in range(T)]; c0=[x>>32 for x in s0]; p0=[x&(B-1) for x in s0]
            q1=(((E[0][1]+O[0][0]+c0[0])&(B-1))*n0inv)&(B-1)
            p1=[0]*T
            for r in range(T):
                c=chain(O[r], [(k,k) for k in range(0,W,2)], nl[r], q1); end(O[r],W,c,1)
                c=chain(E[r], [(k+1,k) for k in range(1,W,2)], nl[r], q1); end(E[r],W+2,c,1)
                s=E[r][1]+O[r][0]+c0[r]; p1[r]=s&(B-1); cin[r]=s>>32
            assert p0[0]==0 and p1[0]==0
            for r in range(T):
                r0=p0[r+1] if r<T-1 else 0; r1=p1[r+1] if r<T-1 else 0
                Z[r]=O[r][1]
                E[r]=E[r][2:]+[0,0]; O[r]=O[r][2:]+[0,0]
                v=E[r][W-2]+(E[r][W-1]<<32)+(E[r][W]<<64)+(E[r][W+1]<<96)+r0+(r1<<32)
                E[r][W-2]=v&(B-1);E[r][W-1]=(v>>32)&(B-1);E[r][W]=(v>>64)&(B-1);E[r][W+1]=(v>>96)&(B-1)
            rnd+=1
    return E,O,Z,cin
def montmul_emu(a,b,n,n0inv, owners=T, W=W):
    E,O,Z,cin=montmul_acc(a,b,n,n0inv,owners,W)
    tot=0
    for r in range(T):
        loc=cin[r]+Z[r]+sum(E[r][k]<<(32*k) for k in range(W+3))+sum(O[r][k]<<(32*(k+1)) for k in range(W+1))
        assert E[r][W+1]==0 and E[r][W+2]==0 and O[r][W-1]==0 and O[r][W]==0 and E[r][W]<=4, (E[r][W:],O[r][W-1:])
        tot+=loc<<(32*W*r)
    return tot
def lanes(x, W=W): return [[(x>>(32*(r*W+j)))&(B-1) for j in range(W)] for r in range(T)]
def value(v): return sum(v[r][j]<<(32*(r*len(v[r])+j)) for r in range(T) for j in range(len(v[r])))
def note(trace, event, lane=None):
    if trace is not None: trace[(event, lane)]+=1
def lane_carry_in(g,p):
    """carry into each lane from per-lane generate / propagate bits, and the carry out of the top lane"""
    c=[0]*T
    for r in range(1,T): c[r]=g[r-1]|(p[r-1]&c[r-1])
    return c, g[T-1]|(p[T-1]&c[T-1])
def group_sub_emu(x,y, trace=None, tag="sub"):
    """d = x - y mod 2^(128 W) over the lanes (x, y as lanes), the borrow out of the top lane"""
    W=len(x[0]); d=[];bo=[]
    for r in range(T):
        v=sum(x[r][j]<<(32*j) for j in range(W))-sum(y[r][j]<<(32*j) for j in range(W))
        bo.append(int(v<0)); d.append([((v%(1<<(32*W)))>>(32*j))&(B-1) for j in range(W)])
    zero=[int(all(l==0 for l in d[r])) for r in range(T)]
    bi,btop=lane_carry_in(bo,zero)
    for r in range(T):
        if bo[r]: note(trace, tag+"_borrow_gen", r)
        if zero[r] and bi[r]: note(trace, tag+"_borrow_prop", r)
        v=(sum(d[r][j]<<(32*j) for j in range(W))-bi[r])%(1<<(32*W)); d[r]=[(v>>(32*j))&(B-1) for j in range(W)]
    return d,btop
def group_ge_emu(x,nl, trace=None):
    W=len(x[0]); gt=[0]*T; lt=[0]*T
    for r in range(T):
        for j in range(W-1,-1,-1):
            if not gt[r] and not lt[r]: gt[r]=int(x[r][j]>nl[r][j]); lt[r]=int(x[r][j]<nl[r][j])
    top=[r for r in range(T) if gt[r] or lt[r]]
    if not top: note(trace, "ge_equal")
    elif top[-1]<T-1: note(trace, "ge_below_top", top[-1])
    return sum(gt[r]<<r for r in range(T))>=sum(lt[r]<<r for r in range(T))
def cond_sub_emu(x,nl, trace=None):
    ge=group_ge_emu(x,nl,trace)
    d,_=group_sub_emu(x,nl,trace,"cond")
    note(trace, "cond_sub_taken" if ge else "cond_sub_skipped")
    return d if ge else x
def mont_finish_emu(E,O,Z,cin,n, W=W, trace=None):
    """mont_finish: merge E, O, Z and the pending carry per lane, carries across the lanes, one subtraction of n on
    overflow.  Returns the W limbs of each lane."""
    v=[];hi=[]
    for r in range(T):
        s=E[r][0]+Z[r]; lim=[s&(B-1)]; c=s>>32
        for k in range(1,W):
            s=E[r][k]+O[r][k-1]+c; lim.append(s&(B-1)); c=s>>32
        h=E[r][W]+O[r][W-1]+c; assert h<B
        v.append(lim); hi.append(h)
    g=[]
    for r in range(T):
        add=(hi[r-1] if r>0 else 0)+cin[r]; assert add<B
        s=sum(v[r][j]<<(32*j) for j in range(W))+add; g.append(s>>(32*W)); v[r]=[(s>>(32*j))&(B-1) for j in range(W)]
    p=[int(all(l==B-1 for l in v[r])) for r in range(T)]
    ci,ctop=lane_carry_in(g,p)
    for r in range(T):
        if g[r]: note(trace, "finish_carry_gen", r)
        if p[r] and ci[r]: note(trace, "finish_carry_prop", r)
        s=(sum(v[r][j]<<(32*j) for j in range(W))+ci[r])%(1<<(32*W)); v[r]=[(s>>(32*j))&(B-1) for j in range(W)]
    if hi[T-1]+ctop!=0:
        note(trace, "finish_overflow")
        v,_=group_sub_emu(v,lanes(n,W),trace,"finish")
    return v
def n0inv_of(n): return (-pow(n,-1,B))%B
def mont_mul_emu(a,b,n, W=W, trace=None, owners=T):
    """mont_mul as K1, K5 and K6a run it: a b R^-1 mod n, almost reduced (< R = 2^(128 W))"""
    return value(mont_finish_emu(*montmul_acc(a,b,n,n0inv_of(n),owners,W),n,W,trace))
def modprod_emu(vals,n, W=W, trace=None, trace_from=None):
    """modprod_kernel (modexp.cuh) for one item: prod(vals) mod n.  Only the products from index `trace_from` on (the
    product with vals[i] for i >= trace_from, default: the last one) and the two closing cond_subs are traced."""
    R=1<<(32*T*W); r2=R*R%n; nl=lanes(n,W)
    tf=len(vals)-1 if trace_from is None else trace_from
    acc=vals[0]
    for i in range(1,len(vals)):
        t=mont_mul_emu(acc,r2,n,W)
        acc=mont_mul_emu(t,vals[i],n,W,trace if i>=tf else None)
    x=cond_sub_emu(lanes(acc,W),nl,trace)
    return value(cond_sub_emu(x,nl,trace))
def check_random(W=W, iters=200, seed=1):
    """random and adversarial products (operands R - 1, modulus R - 1) against big-int arithmetic"""
    random.seed(seed)
    b=32*T*W; R=1<<b
    for it in range(iters):
        n=random.getrandbits(b)|(1<<(b-1))|1
        a=random.getrandbits(b); bb=random.getrandbits(b)
        if it%7==0: a=R-1; bb=R-1
        if it%11==0: n=R-1
        n0inv=(-pow(n,-1,B))%B
        t=montmul_emu(a,bb,n,n0inv,W=W)
        assert t == (a*bb + ((a*bb*(-pow(n,-1,R)))%R)*n)//R
        assert t < R+n
        v=mont_mul_emu(a,bb,n,W)
        assert v < R and v%n == a*bb*pow(R,-1,n)%n
if __name__=="__main__":
    check_random()
    print("emulation ok")
