"""The named configs that stand for the reference's own model configs, pinned to its ymls (TaskPrompter/configs/**,
InvPT/configs/**) and backbone factories, and the batches the float64 suites run them at pinned to the ymls' trBatch /
valBatch. Runs where the reference tree is present (oracle/ref_loader.py) and skips elsewhere; reads the few keys it
needs with a line parser (no YAML library)."""
import os
import re

import pytest

from oracle import configs, ref_loader
from plan_calls import RUNS

pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")

# config name -> (project, yml under <project>/configs/)
YML = {"tp_nyud_vitL": ("TaskPrompter", "nyud/nyud_vitLp16_taskprompter.yml"),
       "tp_pascal_vitB": ("TaskPrompter", "pascal/pascal_vitBp16_taskprompter.yml"),
       "tp_cfg4": ("TaskPrompter", "pascal/pascal_vitLp16_taskprompter.yml"),
       "ip_nyud_vitL": ("InvPT", "nyud/nyud_vitLp16.yml"),
       "ip_cfg3": ("InvPT", "pascal/pascal_vitLp16.yml"),
       "tps_swinB3d": ("TaskPrompter", "cityscapes3d/cs_swinB_taskprompter.yml")}
SCALE = {"PASCALContext": (512, 512), "NYUD": (448, 576)}     # utils/config.py: cfg.TRAIN.SCALE per train_db_name


def _read(project, rel):
    with open(os.path.join(ref_loader.reference_root(), project, rel)) as fh:
        return fh.read()


def yml_keys(text):
    """{key: value string} of every `key: value` line (nesting ignored: the keys read here are unique)."""
    out = {}
    for line in text.splitlines():
        m = re.match(r"\s*([A-Za-z_][\w]*)\s*:\s*([^#]*?)\s*(#.*)?$", line)
        if m and m.group(2):
            out[m.group(1)] = m.group(2).strip("'\"")
    return out


def _tasks(project, keys):
    """The task list in parse_task_dictionary's order (utils/config.py: one `include_<task>` test after another)."""
    order = re.findall(r"'include_(\w+)' in task_dictionary", _read(project, "utils/config.py"))
    return [t for t in order if keys.get(f"include_{t}") == "True"]


def _factory(project, fn):
    """The keyword arguments select_list, embed_dim, depth, num_heads, patch_size of a backbone factory."""
    src = _read(project, "models/transformers/" + ("taskprompter.py" if project == "TaskPrompter" else "vit.py"))
    body = src[src.index(f"def {fn}("):]
    line = re.search(r"model_kwargs = dict\((.*)\)", body).group(1)
    sel = re.search(r"select_list\s*=\s*(range\([^)]*\)|\[[^\]]*\])", line).group(1)
    kw = {k: int(v) for k, v in re.findall(r"(embed_dim|depth|num_heads|patch_size)=(\d+)", line)}
    kw["select"] = list(eval(sel, {"range": range}))
    return kw


@pytest.mark.parametrize("name", [n for n in YML if n.startswith("tp_")])
def test_taskprompter_config_is_the_reference_yml(name):
    project, rel = YML[name]
    k = yml_keys(_read(project, "configs/" + rel))
    cfg = configs.taskprompter(name)
    fn = {"TaskPrompter_vitL": "taskprompter_vit_large_patch16_384",
          "TaskPrompter_vitB": "taskprompter_vit_base_patch16_384"}[k["backbone"]]
    f = _factory(project, fn)
    assert (cfg["C"], cfg["depth"], cfg["heads"], cfg["patch"], cfg["select"]) == \
        (f["embed_dim"], f["depth"], f["num_heads"], f["patch_size"], f["select"])
    assert cfg["tasks"] == _tasks(project, k)
    assert tuple(cfg["img_size"]) == SCALE[k["train_db_name"]]
    assert (cfg["e"], cfg["f"], cfg["chan_nheads"], cfg["prompt_len"]) == \
        (int(k["embed_dim"]), int(k["final_embed_dim"]), int(k["chan_nheads"]), int(k["prompt_len"]))
    assert cfg["use_ctr"] == (k["use_ctr"] == "True") and cfg["head"] == k["head"]


@pytest.mark.parametrize("name", [n for n in YML if n.startswith("ip_")])
def test_invpt_config_is_the_reference_yml(name):
    project, rel = YML[name]
    k = yml_keys(_read(project, "configs/" + rel))
    cfg = configs.invpt(name)
    assert k["backbone"] == "vitL" and k["model"] == "TransformerNet"
    f = _factory(project, "vit_large_patch16_384")
    assert (cfg["C"], cfg["depth"], cfg["heads"], cfg["patch"], cfg["select"]) == \
        (f["embed_dim"], f["depth"], f["num_heads"], f["patch_size"], f["select"])
    assert cfg["tasks"] == _tasks(project, k)
    assert tuple(cfg["img_size"]) == SCALE[k["train_db_name"]]
    assert (cfg["embed_dim"], cfg["pred_const"], cfg["down"]) == \
        (int(k["embed_dim"]), int(k["PRED_OUT_NUM_CONSTANT"]), int(k["mtt_resolution_downsample_rate"]))


def test_slices_are_the_full_configs_but_depth():
    """tp_pascal_vitB_d4 is tp_pascal_vitB with 4 blocks, a prompt level after each of the first three."""
    full, d4 = configs.taskprompter("tp_pascal_vitB"), configs.taskprompter("tp_pascal_vitB_d4")
    strip = lambda c: {k: v for k, v in c.items() if k not in ("name", "depth", "select")}
    assert strip(full) == strip(d4) and (d4["depth"], d4["select"]) == (4, [1, 2, 3])


def test_runs_are_at_the_yml_batches():
    """Every config with a yml runs forward and predict() at its valBatch and trains (where the library trains it)
    at its trBatch."""
    for name, (project, rel) in YML.items():
        k = yml_keys(_read(project, "configs/" + rel))
        val, tr = int(k["valBatch"]), int(k["trBatch"])
        assert (name, val, "predict") in RUNS, (name, val)
        if not name.startswith("tps_"):
            assert (name, val, "forward") in RUNS, (name, val)
        if name.startswith("tp_"):
            assert (name, tr, "train") in RUNS, (name, tr)
