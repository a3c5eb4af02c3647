import collections, csv, subprocess, sys, re, os
rep=sys.argv[1]; kern=sys.argv[2]
out = subprocess.run(["ncu","-i",rep,"--page","source","--csv","--print-source","cuda,sass","-k","regex:"+kern],capture_output=True,text=True).stdout
# function starts per file
root=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),"solo_b200","csrc","")
starts={}
for f in os.listdir(root):
    if not f.endswith((".cuh",".cu")): continue
    L=[]
    for n,l in enumerate(open(root+f),1):
        m=re.match(r"^(?:template.*>\s*)?(?:SB_FN|SB_CFN|SB_FN_BIG|SB_HD|__device__|__global__|static)\s.*?\b(\w+)\s*\(",l)
        if m and not l.startswith(" "): L.append((n,m.group(1)))
    starts[f]=L
def fn(f,ln):
    L=starts.get(f,[]); name="?"
    for n,nm in L:
        if n<=ln: name=nm
        else: break
    return name
cur=None;hdr=None
agg=collections.defaultdict(lambda:[0,0])
for r in csv.reader(out.splitlines()):
    if not r: continue
    if r[0]=="File Path": cur=r[1].split("/")[-1]; continue
    if r[0]=="Line No": hdr=r; continue
    if hdr and cur and r[0] not in ("","...","Function Name"):
        try:
            s=int(r[hdr.index("# Samples")]); ie=int(r[hdr.index("Instructions Executed")]); ln=int(r[0])
        except Exception: continue
        k=(cur,fn(cur,ln)); agg[k][0]+=s; agg[k][1]+=ie
tot=sum(v[0] for v in agg.values()); toti=sum(v[1] for v in agg.values())
for k,v in sorted(agg.items(), key=lambda x:-x[1][0])[:60]:
    print("%-22s %-34s %8d %5.1f%% %12d %5.1f%%"%(k[0],k[1],v[0],100*v[0]/tot,v[1],100*v[1]/toti))
