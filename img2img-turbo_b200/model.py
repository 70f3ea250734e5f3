"""Mirror of src/model.py's importable names.

* make_1step_sched        -> closed-form one-step DDPM (model.py:7-11); the engine fuses the step on device.
* my_vae_encoder_fwd / my_vae_decoder_fwd (model.py:14-54) have no Python body here: the patched VAE forwards
  (skip recording, `sample + skip_conv_i(skip * gamma)`) are part of the libi2it graph (csrc/model.cu).
* download_url            -> same behaviour (model.py:57-73), without tqdm.
"""
import os

from _host import OneStepDDPM


def make_1step_sched():
    return OneStepDDPM()


def my_vae_encoder_fwd(self, sample):
    raise RuntimeError("the patched VAE encoder forward runs inside libi2it (csrc/model.cu: build_vae_encoder)")


def my_vae_decoder_fwd(self, sample, latent_embeds=None):
    raise RuntimeError("the patched VAE decoder forward runs inside libi2it (csrc/model.cu: build_vae_decoder)")


def download_url(url, outf):
    if os.path.exists(outf):
        print(f"Skipping download, {outf} already exists")
        return
    import requests
    print(f"Downloading checkpoint to {outf}")
    response = requests.get(url, stream=True)
    response.raise_for_status()
    tmp = outf + ".part"                      # an interrupted download must never be mistaken for the checkpoint
    with open(tmp, "wb") as f:
        for chunk in response.iter_content(1 << 20):
            f.write(chunk)
    os.replace(tmp, outf)
    print(f"Downloaded successfully to {outf}")
