"""The reference's sample configs and what its full schema reads from them, as fixtures for tests/test_config.py and
tests/test_reference_configs_train_host.py:

  reference_configs.tar.xz         every samples/model_config/*.config and examples/configs/*.config, unmodified
  reference_config_fields.json.xz  per config: the field paths under the guarded sections (test_config.GUARDED) that
                                   are set when the config is parsed with the reference's FULL schema (all of
                                   easy_rec/python/protos/*.proto); every config must parse strictly under it

  python tests/golden/make_reference_configs.py     (needs the reference checkout at /root/reference)"""
import glob
import io
import json
import lzma
import os
import sys
import tarfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from easyrec_b200.config import config_util, proto_loader  # noqa: E402
from test_config import GUARDED, set_field_paths  # noqa: E402

REF = '/root/reference'
RELS = ('samples/model_config', 'examples/configs')


def main():
  paths = [p for d in RELS for p in sorted(glob.glob(os.path.join(REF, d, '*.config')))]
  full = proto_loader.load_schema(sorted(glob.glob(os.path.join(REF, 'easy_rec/python/protos/*.proto'))),
                                  virtual_name='full_ref.proto')
  fields = {}
  with tarfile.open(os.path.join(HERE, 'reference_configs.tar.xz'), 'w:xz', preset=9) as tar:
    for p in paths:
      rel = os.path.relpath(p, REF)
      data = open(p, 'rb').read()
      info = tarfile.TarInfo(rel)
      info.size, info.mode = len(data), 0o644   # mtime 0, no owner: the archive depends on the contents only
      tar.addfile(info, io.BytesIO(data))
      cfg = config_util.get_configs_from_pipeline_file(data, schema=full)   # strict: complete schema
      fields[rel] = sorted(f for f in set_field_paths(cfg) if f.startswith(GUARDED))
  with lzma.open(os.path.join(HERE, 'reference_config_fields.json.xz'), 'wt', preset=9) as f:
    json.dump({'_provenance': 'alibaba/EasyRec @ bd230cb, tests/golden/make_reference_configs.py', 'fields': fields},
              f, indent=0, sort_keys=True)
  print('%d configs' % len(paths))


if __name__ == '__main__':
  main()
