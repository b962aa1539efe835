"""Writes tests/golden/grid_cli/: what `evaluate -useGt -saveRanks` and `generate` write for a grid (pool5) checkpoint of
`mn-att-ques-im-hist + disc` on small synthetic files, in fp32 math (generate answers from the split's answer pool).  The files were made
with the build before region features (DESIGN §26) existed; tests/test_grid_cli_golden_gpu.py runs the same recipe with the
current build and requires the same bytes, so a grid run writes exactly what it wrote before.

usage (from the root of the tree whose build should write the files, on a GPU):
    PYTHONPATH=. python <this file> <out dir>"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

V = 40
SPLITS = {"train": 20, "val": 7}
CASES = [("mn-att-ques-im-hist", "disc")]


def params(enc, dec):
    from visdial_b200.engine import DEFAULT_PARAMS, derive_flags
    p = dict(DEFAULT_PARAMS)
    p.update(encoder=enc, decoder=dec, vocabSize=V, embedSize=12, rnnHiddenSize=32, numLayers=2, imgFeatureSize=8,
             imgSpatialSize=3, imgEmbedSize=8, commonEmbeddingSize=16, numAttentionLayers=1, maxQuesCount=10,
             numOptions=100, dropout=0.5, gpuid=0)
    return derive_flags(p)


def write_inputs(d, p):
    """visdial_params.json / visdial_data.h5 / data_img.h5 (pool5 grid) under d, and the checkpoint model.t7"""
    from visdial_b200 import h5lite
    from visdial_b200.checkpoint import save_checkpoint
    from visdial_b200.model import Model
    from visdial_b200.synthetic import make_corpus
    ques, imgs, info = {}, {}, {"word2ind": {"w%d" % i: i for i in range(1, V - 1)}}
    for i, (split, n) in enumerate(SPLITS.items()):
        raw = make_corpus(p, n, 40, seed=31 + i, max_ques_len=8, max_ans_len=6, max_cap_len=14)
        imgs["images_" + split] = raw.pop("images")
        ques.update({k + "_" + split: np.asarray(v, np.uint32) for k, v in raw.items()})
        info["unique_img_" + split] = ["COCO_%s2014_%012d.jpg" % (split, 1000 * i + j) for j in range(n)]
    h5lite.write(os.path.join(d, "visdial_data.h5"), ques)
    h5lite.write(os.path.join(d, "data_img.h5"), imgs)
    with open(os.path.join(d, "visdial_params.json"), "w") as f:
        json.dump(info, f)
    m = Model(params(p["encoder"], p["decoder"]), seed=5)
    save_checkpoint(m, os.path.join(d, "model.t7"), final=True)
    m.engine.close()


def produce(out_dir, root):
    """runs the recipe with the package under `root`; copies <enc>__<dec>__ranks.json / __results.json into out_dir"""
    os.makedirs(out_dir, exist_ok=True)
    env = dict(os.environ, PYTHONPATH=root)
    for enc, dec in CASES:
        d = tempfile.mkdtemp()
        try:
            write_inputs(d, params(enc, dec))
            files = ["-inputJson", "visdial_params.json", "-inputQues", "visdial_data.h5", "-inputImg", "data_img.h5",
                     "-loadPath", "model.t7", "-math", "fp32"]
            for mod, extra in (("evaluate", ["-useGt", "-saveRanks", "-saveRankPath", "ranks.json", "-batchSize", "4"]),
                               ("generate", ["-maxThreads", "5", "-resultPath", "res"])):
                r = subprocess.run([sys.executable, "-m", "visdial_b200." + mod] + files + extra, cwd=d, env=env,
                                   capture_output=True, text=True, timeout=900)
                assert r.returncode == 0, (mod, r.stdout[-2000:], r.stderr[-2000:])
            tag = "%s__%s__" % (enc, dec)
            shutil.copy(os.path.join(d, "ranks.json"), os.path.join(out_dir, tag + "ranks.json"))
            shutil.copy(os.path.join(d, "res", "results.json"), os.path.join(out_dir, tag + "results.json"))
        finally:
            shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    produce(sys.argv[1], os.getcwd())
