"""TEST-ONLY torch emulation of the kernel the Swin sub-module forwards add to the library (mtt_swin_logit_maps,
include/mtt_b200.h), on top of tests/emul_ops.py's emulation of every other entry point.

`install(monkeypatch)` installs tests/emul_ops.py, then replaces `mtt_b200.ops.swin_logit_maps` with a CPU
restatement that reads and writes the same buffers with the same indexing rule. The product never imports this module.
"""


def install(mp):
    import emul_ops
    from mtt_b200 import ops

    emul_ops.install(mp)

    def swin_logit_maps(logits, maps, *, T, to_maps):
        """logits [.., T + L] (map at column T on) <-> maps [.., H, W]; the first T logit columns are not written."""
        lg = logits.reshape(-1, logits.shape[-1])
        mp_ = maps.reshape(lg.shape[0], -1)
        if to_maps:
            mp_.copy_(lg[:, T:])
        else:
            lg[:, T:] = mp_

    mp.setattr(ops, "swin_logit_maps", swin_logit_maps)
