"""Match the in-graph kernel durations of `bench.py --kineto FILE` to op shapes (read here, no GPU needed).

`FILE.seq` lists the kernels of one graph replay in launch order (CUPTI duration, grid, name); `FILE.ops` lists the
hallo_b200.ops calls of one eager step in the same order.  Every op launches a known set of kernels (a GroupNorm is one
fused launch or three; everything else one), so walking both lists in step gives the warm, in-graph time of every op
shape.
    python tools/kineto_by_shape.py FILE [rows]"""
import re,collections,sys
def load(prefix):
    seq=[l.rstrip('\n') for l in open(prefix+'.seq')]
    ops=[l.rstrip('\n') for l in open(prefix+'.ops')]
    ks=[]
    for l in seq:
        m=re.match(r'\s*([\d.]+) us\s+grid (\[.*?\]|None)\s+(.*)',l)
        ks.append((float(m.group(1)), m.group(2), m.group(3)))
    return ks,ops
EXP={'gemm':['gemm_tc'],'conv3x3':['gemm_tc'],'conv3x3s2':['gemm_tc'],'layernorm':['layernorm'],'attention':['attn_tc'],
     'cross_attention':['xattn','attn_tc'],'temporal_attention':['tattn'],'phase_split':['phase_split'],'upsample2x':['upsample'],
     'timestep_embed':['timestep'],'im2col_latent':['im2col'],'cfg_ddim_step':['cfg_ddim'],'groupnorm':['gn_']}
def align(prefix):
    ks,ops=load(prefix)
    i=0; out=[]
    for op in ops:
        kind=op.split()[0]
        pref=EXP[kind]
        # skip non-matching kernels (torch elementwise, advance_step)
        while i<len(ks) and not any(p in ks[i][2] for p in pref): i+=1
        if kind=='groupnorm':
            t=0; names=[]
            if 'gn_fused' in ks[i][2]:
                t=ks[i][0]; names=[ks[i][2]]; i+=1
            else:
                for _ in range(3):
                    assert 'gn_' in ks[i][2], ks[i]
                    t+=ks[i][0]; names.append(ks[i][2]); i+=1
            out.append((op,t,'+'.join(n.split('<')[0] for n in names),None))
        else:
            out.append((op,ks[i][0],ks[i][2],ks[i][1])); i+=1
    return out
if __name__=='__main__':
    a=align(sys.argv[1])
    agg=collections.OrderedDict()
    for op,t,k,g in a:
        key=(op,k,g)
        c=agg.setdefault(key,[0,0.0]); c[0]+=1; c[1]+=t
    tot=sum(v[1] for v in agg.values())
    print(f"total {tot/1e3:.3f} ms")
    for (op,k,g),(n,t) in sorted(agg.items(), key=lambda kv:-kv[1][1])[:int(sys.argv[2]) if len(sys.argv)>2 else 60]:
        print(f"{t/1e3:7.3f} ms x{n:3d} {t/n:8.1f} us  {op:42s} {g}  {k[:48]}")
