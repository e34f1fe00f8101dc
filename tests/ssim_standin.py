"""A STAND-IN for the reference modules that dropin.install_ssim() touches, written for the tests: modules.commons.ssim
with an `ssim` that raises (so a passing test proves the call went to dsx), and a tasks.tts.fs2 and a usr module that
bind the name at import, as the reference's do.  The task's loss restates FastSpeech2Task's mel losses: the SSIM loss
over frames with any nonzero bin, on (mel + bias) as one-channel images, and the L1 over the same frames."""
import sys
import textwrap

FILES = {
    "modules/__init__.py": "",
    "modules/commons/__init__.py": "",
    "modules/commons/ssim.py": """
        def ssim(img1, img2, window_size=11, size_average=True):
            raise RuntimeError("stand-in ssim: dropin.install_ssim() should have replaced it")
    """,
    "tasks/__init__.py": "",
    "tasks/tts/__init__.py": "",
    "tasks/tts/fs2.py": """
        import torch.nn.functional as F
        from modules.commons.ssim import ssim


        class MelLossTask:
            def __init__(self, mel_loss="ssim:0.5|l1:0.5"):
                self.loss_and_lambda = {k: float(v) for k, v in (t.split(":") for t in mel_loss.split("|"))}

            @staticmethod
            def speech(target):
                return (target.abs().sum(-1, keepdim=True) != 0).float().expand_as(target)

            def ssim_loss(self, out, target, bias=6.0):
                w = self.speech(target)
                s = ssim(out.unsqueeze(1) + bias, target.unsqueeze(1) + bias, size_average=False)
                return ((1 - s) * w).sum() / w.sum()

            def l1_loss(self, out, target):
                w = self.speech(target)
                return (F.l1_loss(out, target, reduction="none") * w).sum() / w.sum()

            def mel_loss(self, out, target):
                total = 0
                for name, lbd in self.loss_and_lambda.items():
                    total = total + lbd * (self.ssim_loss(out, target) if name == "ssim" else self.l1_loss(out, target))
                return total
    """,
    "usr/__init__.py": "",
    "usr/aux_task.py": """
        from modules.commons.ssim import ssim
    """,
}
ROOTS = ("modules", "tasks", "usr")


def _loaded():
    return [n for n in sys.modules if n in ROOTS or n.startswith(tuple(r + "." for r in ROOTS))]


def install_tree(tmp_path, monkeypatch):
    """writes the stand-in under tmp_path and puts it first on sys.path, dropping any other tree's modules"""
    for rel, body in FILES.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(body).lstrip("\n"))
    monkeypatch.syspath_prepend(str(tmp_path))
    for n in _loaded():
        monkeypatch.delitem(sys.modules, n)


def drop_tree():
    for n in _loaded():
        del sys.modules[n]
