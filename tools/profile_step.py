"""One eager train step at the bench workload under torch.profiler: prints the per-kernel CUDA time table (top N rows).

  python tools/profile_step.py [N]      (LO_B, LO_T, LO_IMPL select batch, decode steps, kernels)
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench_support as bs
from latex_ocr_b200.img2seq import Img2SeqModel
from latex_ocr_b200.data import SimpleVocab

B = int(os.environ.get("LO_B", "64")); T = int(os.environ.get("LO_T", "150"))
kern = os.environ.get("LO_IMPL", "tc")
class Cfg:
    encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"; cuda_graph = False
torch.manual_seed(1234)
m = Img2SeqModel(Cfg(), vocab=SimpleVocab(500), device="cuda:0", precision="bf16", impl=kern)
m.build_train(); m.train_mode(True)
img, formula = bs.synthetic_batch(B, 128, 512, 500, T, seed=1234)
img, formula = img.cuda(), formula.cuda()
for _ in range(2):
    m.train_step(img, formula)
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    m.train_step(img, formula)
    torch.cuda.synchronize()
print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=int(sys.argv[1]) if len(sys.argv) > 1 else 25, max_name_column_width=90))
