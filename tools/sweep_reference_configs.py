"""Which reference sample configs build here, and why the others are refused (grouped by message).
Needs /root/reference.   python tools/sweep_reference_configs.py"""
import glob, os, sys, collections, traceback
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
# the plans are built, not trained: tables are allocated but not initialised, and vocabularies get no device index
os.environ.setdefault('ER_PLAN_ONLY', '1')
from easyrec_b200 import builder
from easyrec_b200.config import config_util
REF='/root/reference'
paths = sorted(glob.glob(os.path.join(REF, 'samples/model_config/*.config'))) + sorted(glob.glob(os.path.join(REF, 'examples/configs/*.config')))
ok=[]; errs=collections.defaultdict(list)
for p in paths:
  try:
    cfg = config_util.get_configs_from_pipeline_file(p)
    il, model, opt = builder.build_model(cfg, 8, 'cpu', cpu_generator=torch.Generator().manual_seed(0))
    ok.append(p)
  except Exception as e:
    msg = '%s: %s' % (type(e).__name__, str(e)[:90])
    errs[msg].append(os.path.basename(p))
print('ok', len(ok), 'of', len(paths))
for k,v in sorted(errs.items(), key=lambda kv:-len(kv[1])):
  print(len(v), k, v[:4])
