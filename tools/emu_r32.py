"""Python emulation of the radix-2^32 lane-distributed Montgomery product of
bftkv_b200/csrc/rsa_verify_r32.cuh (same E/O/Z/cin bookkeeping), checked against big-int arithmetic.
`owners` < T stops after that many owner steps, as K1's final check does; mont_finish_emu merges the accumulators and
resolves the carries across the lanes limb for limb (mont_finish), group_sub_emu / cond_sub_emu are group_sub / cond_sub."""
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
def montmul_acc(a,b,n,n0inv, owners=T):
    """the accumulators (E, O, Z, cin) after `owners` owner steps"""
    al=[[ (a>>(32*(r*W+j)))&(B-1) for j in range(W)] for r in range(T)]
    bl=[[ (b>>(32*(r*W+j)))&(B-1) for j in range(W)] for r in range(T)]
    nl=[[ (n>>(32*(r*W+j)))&(B-1) for j in range(W)] for r in range(T)]
    E=[[0]*19 for _ in range(T)]; O=[[0]*17 for _ in range(T)]; cin=[0]*T; Z=[0]*T
    rnd=0
    for owner in range(owners):
        for jj in range(0,W,2):
            b0=bl[owner][jj]; b1=bl[owner][jj+1]
            for r in range(T):
                c=chain(E[r], [(k,k) for k in range(0,W,2)], al[r], b0, cin[r]); end(E[r],16,c,2)
            q0=(((E[0][0]+Z[0])&(B-1))*n0inv)&(B-1)
            for r in range(T):
                c=chain(O[r], [(k-1,k) for k in range(1,W,2)], al[r], b0); end(O[r],16,c,1)
                c=chain(O[r], [(k,k) for k in range(0,W,2)], al[r], b1); end(O[r],16,c,1)
                c=chain(E[r], [(k+1,k) for k in range(1,W,2)], al[r], b1); end(E[r],18,c,1)
                c=chain(E[r], [(k,k) for k in range(0,W,2)], nl[r], q0); end(E[r],16,c,2)
                c=chain(O[r], [(k-1,k) for k in range(1,W,2)], nl[r], q0); end(O[r],16,c,1)
            s0=[E[r][0]+Z[r] for r in range(T)]; c0=[x>>32 for x in s0]; p0=[x&(B-1) for x in s0]
            q1=(((E[0][1]+O[0][0]+c0[0])&(B-1))*n0inv)&(B-1)
            p1=[0]*T
            for r in range(T):
                c=chain(O[r], [(k,k) for k in range(0,W,2)], nl[r], q1); end(O[r],16,c,1)
                c=chain(E[r], [(k+1,k) for k in range(1,W,2)], nl[r], q1); end(E[r],18,c,1)
                s=E[r][1]+O[r][0]+c0[r]; p1[r]=s&(B-1); cin[r]=s>>32
            assert p0[0]==0 and p1[0]==0
            for r in range(T):
                r0=p0[r+1] if r<T-1 else 0; r1=p1[r+1] if r<T-1 else 0
                Z[r]=O[r][1]
                E[r]=E[r][2:]+[0,0]; O[r]=O[r][2:]+[0,0]
                v=E[r][14]+(E[r][15]<<32)+(E[r][16]<<64)+(E[r][17]<<96)+r0+(r1<<32)
                E[r][14]=v&(B-1);E[r][15]=(v>>32)&(B-1);E[r][16]=(v>>64)&(B-1);E[r][17]=(v>>96)&(B-1)
            rnd+=1
    return E,O,Z,cin
def montmul_emu(a,b,n,n0inv, owners=T):
    E,O,Z,cin=montmul_acc(a,b,n,n0inv,owners)
    tot=0
    for r in range(T):
        loc=cin[r]+Z[r]+sum(E[r][k]<<(32*k) for k in range(19))+sum(O[r][k]<<(32*(k+1)) for k in range(17))
        assert E[r][17]==0 and E[r][18]==0 and O[r][15]==0 and O[r][16]==0 and E[r][16]<=4, (E[r][16:],O[r][15:])
        tot+=loc<<(32*W*r)
    return tot
def lanes(x): return [[(x>>(32*(r*W+j)))&(B-1) for j in range(W)] for r in range(T)]
def value(v): return sum(v[r][j]<<(32*(r*W+j)) for r in range(T) for j in range(W))
def lane_carry_in(g,p):
    """carry into each lane from per-lane generate / propagate bits, and the carry out of the top lane"""
    c=[0]*T
    for r in range(1,T): c[r]=g[r-1]|(p[r-1]&c[r-1])
    return c, g[T-1]|(p[T-1]&c[T-1])
def group_sub_emu(x,y):
    """d = x - y mod 2^2048 over the lanes (x, y as lanes), the borrow out of the top lane"""
    d=[];bo=[]
    for r in range(T):
        v=sum(x[r][j]<<(32*j) for j in range(W))-sum(y[r][j]<<(32*j) for j in range(W))
        bo.append(int(v<0)); d.append([((v%(1<<(32*W)))>>(32*j))&(B-1) for j in range(W)])
    bi,btop=lane_carry_in(bo,[int(all(l==0 for l in d[r])) for r in range(T)])
    for r in range(T):
        v=(sum(d[r][j]<<(32*j) for j in range(W))-bi[r])%(1<<(32*W)); d[r]=[(v>>(32*j))&(B-1) for j in range(W)]
    return d,btop
def group_ge_emu(x,nl):
    gt=[0]*T; lt=[0]*T
    for r in range(T):
        for j in range(W-1,-1,-1):
            if not gt[r] and not lt[r]: gt[r]=int(x[r][j]>nl[r][j]); lt[r]=int(x[r][j]<nl[r][j])
    return sum(gt[r]<<r for r in range(T))>=sum(lt[r]<<r for r in range(T))
def cond_sub_emu(x,nl):
    d,_=group_sub_emu(x,nl)
    return d if group_ge_emu(x,nl) else x
def mont_finish_emu(E,O,Z,cin,n):
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
    ci,ctop=lane_carry_in(g,[int(all(l==B-1 for l in v[r])) for r in range(T)])
    for r in range(T):
        s=(sum(v[r][j]<<(32*j) for j in range(W))+ci[r])%(1<<(32*W)); v[r]=[(s>>(32*j))&(B-1) for j in range(W)]
    if hi[T-1]+ctop!=0:
        v,_=group_sub_emu(v,lanes(n))
    return v
if __name__=="__main__":
    random.seed(1)
    R=1<<2048
    for it in range(200):
        n=random.getrandbits(2048)|(1<<2047)|1
        a=random.getrandbits(2048); b=random.getrandbits(2048)
        if it%7==0: a=R-1; b=R-1
        if it%11==0: n=R-1
        n0inv=(-pow(n,-1,B))%B
        t=montmul_emu(a,b,n,n0inv)
        assert t == (a*b + ((a*b*(-pow(n,-1,R)))%R)*n)//R
        assert t < R+n
    print("emulation ok")
