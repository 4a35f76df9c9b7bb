"""Named model configurations: the reference's yml model blocks as plain dicts (synthetic shapes per SURVEY.md section 8d / BASELINE.json configs).

Data only: shared by the bench, the tests and the CPU oracle."""

PASCAL_TASKS = ["semseg", "human_parts", "sal", "normals", "edge"]
PASCAL_OUT = {"semseg": 21, "human_parts": 7, "sal": 2, "normals": 3, "edge": 1}
NYUD_TASKS = ["semseg", "depth", "normals", "edge"]
NYUD_OUT = {"semseg": 40, "depth": 1, "normals": 3, "edge": 1}


def taskprompter(name):
    """Config dicts for TaskPrompter (TP/models/transformers/taskprompter.py:285-366)."""
    c = {
        # tiny models for golden fixtures / CPU tests
        "tp_tiny": dict(tasks=["semseg", "depth", "normals"], num_output={"semseg": 5, "depth": 1, "normals": 3},
                        img_size=(64, 96), patch=16, C=128, depth=4, heads=2, select=[1, 2, 3],
                        e=24, f=32, chan_nheads=4, use_ctr=True),
        "tp_tiny1": dict(tasks=["semseg", "edge"], num_output={"semseg": 4, "edge": 1},
                         img_size=(64, 64), patch=16, C=128, depth=4, heads=2, select=[1, 2, 3],
                         e=20, f=28, chan_nheads=1, use_ctr=False),
        # DEConvHead heads (taskprompter.py:700-715; `head: deconv`, the Cityscapes-3D yml) on a tiny ViT backbone
        "tp_tiny_de": dict(tasks=["semseg", "depth"], num_output={"semseg": 6, "depth": 1},
                           img_size=(64, 96), patch=16, C=128, depth=4, heads=2, select=[1, 2, 3],
                           e=24, f=32, chan_nheads=1, use_ctr=False, head="deconv"),
        # BASELINE.json configs[1]: ViT-B geometry + NYUD decoder dims (SURVEY.md section 0 row 4)
        "tp_cfg2": dict(tasks=NYUD_TASKS, num_output=NYUD_OUT, img_size=(448, 576), patch=16, C=768, depth=12,
                        heads=12, select=[3, 6, 9], e=768, f=768, chan_nheads=16, use_ctr=False),
        # BASELINE.json configs[3]: TaskPrompter ViT-L PASCAL-Context, the headline metric's config
        "tp_cfg4": dict(tasks=PASCAL_TASKS, num_output=PASCAL_OUT, img_size=(512, 512), patch=16, C=1024,
                        depth=24, heads=16, select=[6, 12, 18], e=300, f=350, chan_nheads=1, use_ctr=True),
        # a 2-block slice of cfg4 geometry for full-size kernel parity at low cost
        "tp_cfg4_d4": dict(tasks=PASCAL_TASKS, num_output=PASCAL_OUT, img_size=(512, 512), patch=16, C=1024,
                           depth=4, heads=16, select=[1, 2, 3], e=300, f=350, chan_nheads=1, use_ctr=True),
        # a 4-block slice of cfg2 geometry (4 x 4 channel windows, e = f = 768, no ctr) for the reverse pass at full width
        "tp_cfg2_d4": dict(tasks=NYUD_TASKS, num_output=NYUD_OUT, img_size=(448, 576), patch=16, C=768, depth=4,
                           heads=12, select=[1, 2, 3], e=768, f=768, chan_nheads=16, use_ctr=False),
        # BASELINE.json configs[4] stand-in (SURVEY.md section 0 row 5)
        "tp_cfg5": dict(tasks=["semseg", "depth", "3ddet"], num_output={"semseg": 19, "depth": 1, "3ddet": 18},
                        img_size=(1024, 2048), patch=16, C=1024, depth=24, heads=16, select=[6, 12, 18],
                        e=300, f=350, chan_nheads=1, use_ctr=False),
        # the reference's own model configs (TP/configs/nyud/nyud_vitLp16_taskprompter.yml and
        # TP/configs/pascal/pascal_vitBp16_taskprompter.yml; select from taskprompter.py:675 / :683)
        "tp_nyud_vitL": dict(tasks=NYUD_TASKS, num_output=NYUD_OUT, img_size=(448, 576), patch=16, C=1024, depth=24,
                             heads=16, select=[6, 12, 18], e=768, f=768, chan_nheads=16, use_ctr=False),
        "tp_pascal_vitB": dict(tasks=PASCAL_TASKS, num_output=PASCAL_OUT, img_size=(512, 512), patch=16, C=768,
                               depth=12, heads=12, select=[3, 6, 9], e=780, f=1024, chan_nheads=16, use_ctr=True),
        # a 4-block slice of tp_pascal_vitB (4 x 4 channel windows with ctr, e = 780, f = 1024) for the reverse pass
        "tp_pascal_vitB_d4": dict(tasks=PASCAL_TASKS, num_output=PASCAL_OUT, img_size=(512, 512), patch=16, C=768,
                                  depth=4, heads=12, select=[1, 2, 3], e=780, f=1024, chan_nheads=16, use_ctr=True),
        # long, non-square sequence (N = 2 + 16*128 = 2050 tokens) at ViT-L width: cheap stand-in for cfg5 in tests
        "tp_long": dict(tasks=["semseg", "depth"], num_output={"semseg": 19, "depth": 1},
                        img_size=(256, 2048), patch=16, C=1024, depth=4, heads=16, select=[1, 2, 3],
                        e=300, f=350, chan_nheads=4, use_ctr=False),
        # 4-block slice of the cfg5 geometry (N = 8195 tokens) for long-sequence parity at tractable oracle cost
        "tp_cfg5_d4": dict(tasks=["semseg", "depth", "3ddet"], num_output={"semseg": 19, "depth": 1, "3ddet": 18},
                           img_size=(1024, 2048), patch=16, C=1024, depth=4, heads=16, select=[1, 2, 3],
                           e=300, f=350, chan_nheads=1, use_ctr=False),
    }[name]
    c = dict(c)
    c["name"] = name
    c["prompt_len"] = 1
    c.setdefault("head", "conv")     # utils/common_config.py:64-70: 'conv' -> ConvHead, 'deconv' -> DEConvHead
    return c


def taskprompter_swin(name):
    """Config dicts for the Swin TaskPrompter (TP/models/transformers/taskprompter_swin.py:542-666, built by
    TP/utils/common_config.py:34-41): SURVEY.md section 8f N2. Only the CPU oracle uses them so far."""
    c = {
        # tiny: 64x96 image, patch 4 -> 16x24 tokens, four stages (levels 8x12 / 4x6 / 2x3 / 2x3 after merging); window 4
        # with shifted windows in the first stages, then windows clipped to the map and PADDED (2x3 -> 2x4)
        "tps_tiny": dict(tasks=["semseg", "depth"], num_output={"semseg": 5, "depth": 1}, img_size=(64, 96), patch=4,
                         embed_dim=16, depths=(2, 2, 2, 2), heads=(1, 2, 4, 8), window=4, img_ds_ratio=1.0,
                         level_embed_dim=12, f=24, chan_embed_dim=16, chan_nheads=1, head="deconv"),
        # 64x128 image (levels 8x16 / 4x8 / 2x4 / 2x4), 2x2 channel-attention windows, ConvHead, three tasks
        "tps_tiny4": dict(tasks=["semseg", "depth", "normals"], num_output={"semseg": 4, "depth": 1, "normals": 3},
                          img_size=(64, 128), patch=4, embed_dim=16, depths=(2, 2, 2, 2), heads=(2, 2, 4, 4), window=4,
                          img_ds_ratio=1.0, level_embed_dim=10, f=20, chan_embed_dim=16, chan_nheads=4, head="conv"),
        # the reference config's window (12, shift 6), input down-scaling (0.75) and dd_label_map_size at toy width:
        # 256x512 -> 192x384 -> tokens 48x96 / 24x48 / 12x24 (window clipped to 12) / 6x12 (window 6)
        "tps_mid": dict(tasks=["semseg", "depth"], num_output={"semseg": 19, "depth": 1}, img_size=(256, 512), patch=4,
                        embed_dim=16, depths=(2, 2, 2, 2), heads=(1, 2, 4, 8), window=12, img_ds_ratio=0.75,
                        level_embed_dim=16, f=24, chan_embed_dim=16, chan_nheads=1, head="deconv",
                        dd_label_map_size=(128, 256)),
        # the reference's Cityscapes-3D model (cs_swinB_taskprompter.yml) without the 3ddet task
        "tps_swinB": dict(tasks=["semseg", "depth"], num_output={"semseg": 19, "depth": 1}, img_size=(1024, 2048),
                          patch=4, embed_dim=128, depths=(2, 2, 18, 2), heads=(4, 8, 16, 32), window=12,
                          img_ds_ratio=0.75, level_embed_dim=256, f=450, chan_embed_dim=256, chan_nheads=1,
                          head="deconv", dd_label_map_size=(512, 1024)),
        # ---- three tasks with '3ddet' (its detection head is the caller's module; num_output["3ddet"] only sizes the
        # oracle's dense stand-in parameters, which the fixtures drop)
        # tiny: 64x128, window 6 (shift 3) padded to 18x36 / 12x18, then clipped to 4 and 2; 2x2 channel windows
        "tps_tiny3d": dict(tasks=["semseg", "depth", "3ddet"], num_output={"semseg": 5, "depth": 1, "3ddet": 1},
                           img_size=(64, 128), patch=4, embed_dim=16, depths=(2, 2, 2, 2), heads=(1, 2, 4, 8), window=6,
                           img_ds_ratio=1.0, level_embed_dim=12, f=24, chan_embed_dim=16, chan_nheads=4, head="deconv"),
        # tps_mid with the 3ddet task: window 12, 0.75 input scaling, dd_label_map_size
        "tps_mid3d": dict(tasks=["semseg", "depth", "3ddet"], num_output={"semseg": 19, "depth": 1, "3ddet": 1},
                          img_size=(256, 512), patch=4, embed_dim=16, depths=(2, 2, 2, 2), heads=(1, 2, 4, 8), window=12,
                          img_ds_ratio=0.75, level_embed_dim=16, f=24, chan_embed_dim=16, chan_nheads=1, head="deconv",
                          dd_label_map_size=(128, 256)),
        # the reference's Cityscapes-3D model exactly (cs_swinB_taskprompter.yml: semseg, depth, 3ddet)
        "tps_swinB3d": dict(tasks=["semseg", "depth", "3ddet"], num_output={"semseg": 19, "depth": 1, "3ddet": 1},
                            img_size=(1024, 2048), patch=4, embed_dim=128, depths=(2, 2, 18, 2), heads=(4, 8, 16, 32),
                            window=12, img_ds_ratio=0.75, level_embed_dim=256, f=450, chan_embed_dim=256, chan_nheads=1,
                            head="deconv", dd_label_map_size=(512, 1024)),
    }[name]
    c = dict(c)
    c["name"] = name
    c["prompt_len"] = 1
    return c


def invpt(name):
    """Config dicts for InvPT (IP/models/transformer_net.py, IP/utils/common_config.py:15-51)."""
    c = {
        # BASELINE.json configs[0]: ViT-tiny, 2 tasks, 128x128, bs 2
        "ip_cfg1": dict(tasks=["semseg", "depth"], num_output={"semseg": 40, "depth": 1}, img_size=(128, 128),
                        patch=16, C=192, depth=12, heads=3, select=[3, 6, 9], embed_dim=64, pred_const=16,
                        down=2),
        "ip_tiny": dict(tasks=["semseg", "normals"], num_output={"semseg": 6, "normals": 3}, img_size=(64, 128),
                        patch=16, C=128, depth=4, heads=2, select=[1, 2, 3], embed_dim=48, pred_const=16,
                        down=2),
        # BASELINE.json configs[2]: InvPT ViT-L PASCAL-Context
        "ip_cfg3": dict(tasks=PASCAL_TASKS, num_output=PASCAL_OUT, img_size=(512, 512), patch=16, C=1024,
                        depth=24, heads=16, select=[6, 12, 18], embed_dim=512, pred_const=64, down=2),
        # the reference's NYUD model (IP/configs/nyud/nyud_vitLp16.yml; select from IP vit.py:560)
        "ip_nyud_vitL": dict(tasks=NYUD_TASKS, num_output=NYUD_OUT, img_size=(448, 576), patch=16, C=1024,
                             depth=24, heads=16, select=[6, 12, 18], embed_dim=512, pred_const=64, down=2),
    }[name]
    c = dict(c)
    c["name"] = name
    return c
