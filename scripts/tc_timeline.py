"""Diagnostic: clock64 timeline of CTA (0,0) of the LAST wgmma conv launch of an eval iteration
(MAML_B200_TC_TIMELINE=1, graphs off).  Marks: 0 start, 1 setup done (barriers, row flags), 2 first A tile landed,
3 first B stage landed, 4 B stage 9 landed, 5 last MMA complete, 6 both warpgroups done (tile overwrites operands),
7 epilogue rows stored / pushed, 10-12 (split-K) after the cluster
barrier, the reduction, the statistics, 8 epilogue done."""
import os, sys
os.environ["MAML_B200_TC_TIMELINE"] = sys.argv[3] if len(sys.argv) > 3 else "0"     # block to record (0 = any)
os.environ["MAML_B200_NO_GRAPH"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier, make_args, synthetic_batch
name = sys.argv[1] if len(sys.argv) > 1 else "omniglot_mamlpp_5w1s"
mode = sys.argv[2] if len(sys.argv) > 2 else "eval"
dev = torch.device("cuda", 0)
a = make_args(name)
m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device=dev, args=a)
b = synthetic_batch(a, 0)
db = (b[0].to(dev), b[1].to(dev), b[2].long().to(dev), b[3].long().to(dev))
for _ in range(3):
    m._run(db, 0, mode == "train", False)
torch.cuda.synchronize()
t = m._engine.debug_read("tc_timeline")
print(name, mode, "block", os.environ["MAML_B200_TC_TIMELINE"], "cycles since start:", [int(x) for x in t[:13]])
