"""The package, the drop-in and the oracle against what the reference itself computed and declares.

tests/golden/reference_diffnet.npz (oracle/gen_golden.py --reference-diffnet) holds one evaluation of the reference's own
DiffNet, its parameter names / shapes, and the state-dict surface of its GaussianDiffusion as the task files build it; the
drop-in is installed into the stand-in tree of tests/standin_ref.py (the reference's module paths and class names)."""
import os
import subprocess
import sys

import numpy as np
import torch

from conftest import HP, ROOT, golden


def test_package_and_oracle_match_reference_fixture(lib_built):
    from diffsinger_b200.modules import DiffNet
    from oracle import diffnet_oracle as O
    g = golden("reference_diffnet.npz")
    torch.manual_seed(0)                                  # the reference's init stream under the same seed
    net = DiffNet(80, hparams=dict(HP, dilation_cycle_length=1))
    torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    sd = net.state_dict()
    assert list(sd.keys()) == [str(k) for k in g["keys"]]
    assert [",".join(map(str, v.shape)) for v in sd.values()] == [str(s) for s in g["shapes"]]
    x, cond, t = (torch.from_numpy(g[k]) for k in ("x", "cond", "t"))
    with torch.no_grad():
        eps = O.diffnet_forward({k: v.detach() for k, v in sd.items()}, x, t, cond, 1)
    # the fixture was bit-exact on the machine that wrote it; other CPUs may pick other conv kernels
    assert np.abs(eps.numpy() - g["eps"]).max() < 1e-5

SCRIPT = r"""
import sys, numpy as np, torch
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests"); sys.path.insert(0, %(tree)r)
from conftest import HP, golden
from oracle import diffnet_oracle as O
from utils.hparams import hparams
g = golden("reference_diffnet.npz")
hparams.update(HP, spec_min=[float(v) for v in g["gd_spec_min"]], spec_max=[float(v) for v in g["gd_spec_max"]],
               schedule_type=str(g["gd_schedule_type"]), max_beta=float(g["gd_max_beta"]), diff_decoder_type="wavenet")
import usr.diff.shallow_diffusion_tts as sdt, usr.diff.net as net_mod
ref_cls, ref_net = sdt.GaussianDiffusion, net_mod.DiffNet
import diffsinger_b200.dropin as dropin
new_cls = dropin.install()
assert sdt.GaussianDiffusion is new_cls and issubclass(new_cls, ref_cls)
assert net_mod.DiffNet.__module__.startswith("diffsinger_b200")

def build():
    # the task files build the model exactly like this (usr/diffspeech_task.py:25-32)
    torch.manual_seed(0)
    return sdt.GaussianDiffusion(phone_encoder=None, out_dims=80, denoise_fn=net_mod.DiffNet(hparams["audio_num_mel_bins"]),
                                 timesteps=int(g["gd_timesteps"]), K_step=int(g["gd_K_step"]), loss_type="l1",
                                 spec_min=hparams["spec_min"], spec_max=hparams["spec_max"])

# checkpoint surface: every entry of the reference module outside its FastSpeech2 conditioner (the stand-in has none),
# same names and shapes, and a checkpoint with exactly those entries loads with strict=True
model = build()
ref_shapes = {str(k): tuple(int(d) for d in str(s).split(",") if d) for k, s in zip(g["gd_keys"], g["gd_shapes"])
              if not str(k).startswith("fs2.")}
assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == ref_shapes
model.load_state_dict({k: torch.zeros(s) for k, s in ref_shapes.items()}, strict=True)
# same init stream as the reference: the installed DiffNet under seed 0 computes the reference's own eps (via the oracle)
model = build()
net = model.denoise_fn
torch.nn.init.normal_(net.output_projection.weight, std=0.02)
x, cond, t = (torch.from_numpy(g[k]) for k in ("x", "cond", "t"))
with torch.no_grad():
    eps = O.diffnet_forward({k: v.detach() for k, v in net.state_dict().items()}, x, t, cond, 1)
assert np.abs(eps.numpy() - g["eps"]).max() < 1e-5
# training branch unchanged: the module graph under autograd, same function
net.train()
out = net(x, t, cond)
assert out.requires_grad and np.abs(out.detach().numpy() - g["eps"]).max() < 1e-5
net.eval()
# the inference branch has no CPU fallback
class Stub(torch.nn.Module):
    def forward(self, *a, **k):
        return {"decoder_inp": torch.randn(2, 24, 256), "mel_out": torch.randn(2, 24, 80)}
model.fs2 = Stub()
try:
    with torch.no_grad():
        model(torch.zeros(2, 5, dtype=torch.long), infer=True)
    raise SystemExit("expected DsxError on CPU")
except Exception as e:
    assert type(e).__name__ == "DsxError", repr(e)
dropin.uninstall()
assert sdt.GaussianDiffusion is ref_cls and net_mod.DiffNet is ref_net
print("LIVE-OK")
"""


def test_dropin_against_live_reference(lib_built, tmp_path):
    from standin_ref import write_tree
    tree = write_tree(str(tmp_path / "standin"))
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    r = subprocess.run([sys.executable, "-c", SCRIPT % {"root": ROOT, "tree": tree}], capture_output=True, text=True, env=env,
                       cwd=ROOT, timeout=600)
    assert "LIVE-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
