import sys, os, time, numpy as np, torch
R=os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0,R); sys.path.insert(0,os.path.join(R,'tests'))
import art_planner_b200 as ap
from art_planner_b200 import synth, costnet
import cases
from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer
import torch.nn.functional as F
m = cases.c4_map()
chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0); chk.setMap(m); chk.updateHeightField()
obj = ap.MotionCostObjective(chk); sd = costnet.make_state_dict(5); obj.setWeights(sd)
for mode in (0, 1):
    obj.setMode(mode)
    ts=[]
    for i in range(6):
        obj.updateFeatures(); ts.append(obj.lastTrunkTimesMs())
    print('mode',mode,'trunk times ms (3x3 stack, 15x15, total):', np.round(np.array(ts[2:]).mean(0),4))
obj.setMode(0); obj.updateFeatures()
q = torch.from_numpy(costnet.make_queries(m, 4096, 6)).cuda(); out=torch.empty((4096,3),device='cuda')
for _ in range(3): obj.costQuery(q,out)
torch.cuda.synchronize(); s=torch.cuda.Event(enable_timing=True); e=torch.cuda.Event(enable_timing=True); s.record()
for _ in range(100): obj.costQuery(q,out)
e.record(); torch.cuda.synchronize(); print('head 4096 queries ms:', s.elapsed_time(e)/100)
# reference-style PyTorch fp16 on GPU (functional restatement = same cuDNN calls as the module)
orc = CostNetOracle(sd)
for dt in (torch.float16, torch.float32):
    orc.p = {k: v.cuda().to(dt) for k,v in orc.p.items()}
    E = torch.as_tensor(cnn_input_from_layer(m.elevation)).cuda().to(dt)
    def feats():
        t=E[None,None]
        t=orc._conv_bn(t,'init_conv1','init_conv1_bn'); t=F.leaky_relu(orc._conv_bn(t,'init_conv2','init_conv2_bn'),0.3); t=F.max_pool2d(t,(2,2),stride=2)
        t=F.leaky_relu(orc._conv_bn(t,'init_conv3','init_conv3_bn'),0.3); t=F.leaky_relu(orc._conv_bn(t,'init_conv4','init_conv4_bn'),0.3); t=F.max_pool2d(t,(3,3),stride=1)
        t=F.leaky_relu(orc._conv_bn(t,'init_conv5','init_conv5_bn'),0.3); t=F.leaky_relu(orc._conv_bn(t,'init_flatten','init_flatten_bn'),0.3); return t
    with torch.no_grad():
        for _ in range(5): feats()
        torch.cuda.synchronize(); s.record()
        for _ in range(20): f=feats()
        e.record(); torch.cuda.synchronize()
    print('torch', dt, 'trunk ms:', s.elapsed_time(e)/20)
