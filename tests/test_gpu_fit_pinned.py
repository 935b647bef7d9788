"""The default fit, pinned bit for bit: SHA-256 of tril(L), alpha, the LML and y statistics (y_mean, y_std, y_opt), the
suggestion over 4096 candidates (index and the bits of value, mu, std), and W for FP64 fits — `digests` in _fit_scale.py — on
cfg3's θ of record (Matérn-5/2, D = 32), FP64 and tensor-core fits.  A tensor-core fit is lazy: its L and alpha are hashed
before anything forms the rest of W.

  N = 700    below the early start on the Gram matrix's first column block (N >= 1024)
  N = 1500   plain priority streams (the SM partition starts at N = 2048)
  N = 2304   the partitioned schedule, 9 panels
  N = 4096   16 panels
  N = 5800   23 panels: an odd count ends the merged bulk pairs early, and the last panel is 168 columns wide
  N = 8192   32 panels

The digests were recorded on one NVIDIA H100 80GB HBM3 at a 700 W power limit (driver 580.159.03), with the library as it was
before the factorisation's alternative schedules (v2, other panel widths and depths, MID rows, the late start) were removed.
They were the same in repeated processes and with KBO_FIT_NO_PARTITION=1, which is checked here too.
"""
import json
import os
import subprocess
import sys

import pytest

from tests import _fit_scale as H

pytestmark = pytest.mark.gpu

HELPER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_fit_scale.py")

PINNED = {
    (700, "f64"): dict(
        L="045ba6eb69d31cb42d16cd7a176c14fdf404212e7b9376d4b35afe8d15c518ed",
        alpha="bb4f2b32f37095a54cd2d1d829fbe43d848d49c98d434eebcb784218b650ec78",
        fit="7a615cd558c71ef258b0002f08f6c672118e71d75aa7c42dcf440bc978def6f8",
        ask="579e0a1f19506cf93c708c0f47dc34a7a313b8b9655167247792c7e63f7ab06a",
        W="89d42b128ece39a12fea8749d14520b3ca72e07eb9b656efaa2291800cbe905a",
    ),
    (700, "tc"): dict(
        L="045ba6eb69d31cb42d16cd7a176c14fdf404212e7b9376d4b35afe8d15c518ed",
        alpha="bb4f2b32f37095a54cd2d1d829fbe43d848d49c98d434eebcb784218b650ec78",
        fit="7a615cd558c71ef258b0002f08f6c672118e71d75aa7c42dcf440bc978def6f8",
        ask="01c0c69021e22f15f3112030a10eeb893cac87cfc8f5f4d96e108c49d4a6230d",
    ),
    (1500, "f64"): dict(
        L="de9bcc3a4cbf6d7bd7b5ff51df84fac081f2e8a9ab450faa0f6a37f185eaca7f",
        alpha="821ea117130141d9f20a37130bb149f6ff2566ced368a51282bcb40add490c41",
        fit="8beb137bf27348f4655feedb5e39388dd4588f65bbba37f1e407c9f7d6f95eea",
        ask="5a112efa80d4e5fa1bca950c46ac0480dddb794234b07e10efb2a372ebc64367",
        W="f86fd9eb9d157130b29856efc8a7cafbea7895d76fda2b1fda7ad137c07d5957",
    ),
    (1500, "tc"): dict(
        L="de9bcc3a4cbf6d7bd7b5ff51df84fac081f2e8a9ab450faa0f6a37f185eaca7f",
        alpha="45b639c87986bff4158f797fce54dcaa388e89138231ad7736602761a615efab",
        fit="3f2539123dcb1a338c966c2cdb9aea2b6ddbec06f3bd4ce17975b61f45c8d117",
        ask="2f68994ffa7d2f93a6da12c2a2a10de18e6d008a62a71630cf5993e2ba68ce5e",
    ),
    (2304, "f64"): dict(
        L="f599f85078fba981bb945d51a75651b67423a94f67cedf9df93c1b0dace9991e",
        alpha="7dec33857f6b2bae387062f244b935cdaba8b510f3adb098592bf64f88b46752",
        fit="abe3d1140b2ca0824a6964e480ff826e1d7178064eaff105e8f18b9770d76545",
        ask="5822407d4c327183cbe8100b85004d49ed5462d2118513d3e54f0ee410f3d39b",
        W="b2042745a871670244ba35236f3b6083aa28d8b9af04a86931a6cce7be133fdd",
    ),
    (2304, "tc"): dict(
        L="f599f85078fba981bb945d51a75651b67423a94f67cedf9df93c1b0dace9991e",
        alpha="be969f9801fce81f99b5078c7f11d796bf323d1aa5ab3650d53d431ea911152d",
        fit="abe3d1140b2ca0824a6964e480ff826e1d7178064eaff105e8f18b9770d76545",
        ask="afc0a86707558b80b7560e7200864fdc3d2e98df020ffd0b122fd2637c26da12",
    ),
    (4096, "f64"): dict(
        L="cb9dc41f72ea186b954677afb82f2c81d810d01c0db7f43a15ed0346f26d4526",
        alpha="e93d622bfc8cb9817ec9627e849cb3a52bb3d1f22c027f8adf1cb225fd8c9156",
        fit="7f2a163135a106697c991e4d5223647ac84e8395eb112290c5d05a941f186aa3",
        ask="18704a10f9f47f461d3052326137eebb1149b45a545d9a6685b33ae3768526e9",
        W="c5ac1b5d260aebff42cf69c23aa23186de5ec1c9361264c15a966423c45486e1",
    ),
    (4096, "tc"): dict(
        L="cb9dc41f72ea186b954677afb82f2c81d810d01c0db7f43a15ed0346f26d4526",
        alpha="2aba64c0178c4fc3ad461934d72d37a78d04da5a8e9e5c8e1c5f61bd78a9ee76",
        fit="7f2a163135a106697c991e4d5223647ac84e8395eb112290c5d05a941f186aa3",
        ask="8c64631b4774d2ed7f25e20e0fa7751f00f98907f1bfbdafc39e0338374a05ca",
    ),
    (5800, "f64"): dict(
        L="81406be5e3601481b006738e10e5244420c1f81e02193633f1cee96ca63a87fe",
        alpha="ab4f9aafe1046a3b2b126941e1bb1bcee4d793919d6728c81d75e7ef51bc01bc",
        fit="e3aecc7fdd7119ea89a37f2c3ca8c160a7c44b32cdeea8390ec97c5687723393",
        ask="eea071ba2898c20ed881462d59cf8b29613af130080378e3f692b942117e7ecb",
        W="dbcb4601b2c141d05c89123b3496fb89ed1eee40f7bccf8c8a5e089f777fc9b1",
    ),
    (5800, "tc"): dict(
        L="81406be5e3601481b006738e10e5244420c1f81e02193633f1cee96ca63a87fe",
        alpha="0806f202f275436137e2fc386271361a8f694dab0c2594efddc89895a6727c77",
        fit="e3aecc7fdd7119ea89a37f2c3ca8c160a7c44b32cdeea8390ec97c5687723393",
        ask="23101a40f7bfbf901d5411baa55504103f09a9465329fbeb3ed1d0b206e8a296",
    ),
    (8192, "f64"): dict(
        L="084132a2e9fd52058bac5bb52bebcb37c73cdce154cf0ac0b93e8d0d2587454b",
        alpha="243c2c9f706397a467a163a22af15a41eaecd9594ca9e29710edf0d9558f29bc",
        fit="bec19c58146accb0c012134945d93871e9b04f57a19a87d2a645616729254f07",
        ask="3692fb0d2eaa262670f64a61c1625bcf1c0ccc272d8be6a85bf26a470db7ac74",
        W="5d5ee572cf441f0b2454f2236bc53e798c38416832ecb1aadd2f44c1940f2a8e",
    ),
    (8192, "tc"): dict(
        L="084132a2e9fd52058bac5bb52bebcb37c73cdce154cf0ac0b93e8d0d2587454b",
        alpha="abacddbf1ab5696a9250edbf7edf75bfe0a544eef6e006bc2684cfda72236548",
        fit="0f14ec8b53fa087ca2f1a356a380e962e0ceb6b1a00d1800f991815a1b93dff8",
        ask="dccc66dc7ebe08d06f58c66da31a35579fb38b523bac7aa73cdb0ec03a6ae0d4",
    ),
}


@pytest.mark.parametrize("N,var_mode", list(PINNED))
def test_default_fit_matches_its_pinned_digests(N, var_mode):
    assert H.digests(N, var_mode) == PINNED[(N, var_mode)]


def test_fit_on_plain_priority_streams_matches_the_pinned_digests(tmp_path):
    """The same schedule with KBO_FIT_NO_PARTITION=1 (read once per process: a fresh one) gives the same bits."""
    out = tmp_path / "digests.json"
    spec = {"digests": [[N, vm] for N, vm in PINNED]}
    subprocess.run([sys.executable, HELPER, json.dumps(spec), str(out)], check=True, env={**os.environ, "KBO_FIT_NO_PARTITION": "1"},
                   timeout=900)
    with open(out) as f:
        got = json.load(f)
    for key, g in zip(PINNED, got):
        assert g == PINNED[key], key
