"""Byte stability of both HEVC encoders: the md5 of every access unit below is pinned.

The host encoder generates every synthetic test stream and the bench.py workload, and the GPU encoder's streams are what
its users store, so a change to the entropy-coding code both share (b200_hevc_enc_cabac.h) must leave their bytes as they
are.  The host cases cover SAO, sign hiding, transform skip, PCM, transquant bypass, scaling lists, tiles, slices,
dependent slice segments, 4:0:0 / 4:2:2 / 4:4:4 and 8 to 12 bits."""
import hashlib

import pytest

from hevc_cases import SYNTH, SYNTH_CPU_EXTRA, synth_stream
from libheif_b200 import hevc_enc

# the bench.py workload tile (make_tile): 1024 x 1024, 8-bit 4:2:0, QP 27, WPP, VUI; seeds 0xB200 + idx
BENCH_TILES = [(0, 5), (3, 5), (17, 5), (0, 6), (9, 6)]


def _vui():
    return dict(vui_present=1, colour_description_present=1, colour_primaries=1, transfer_characteristics=13,
                matrix_coefficients=6, full_range=0)


def host_au(name):
    if name.startswith("smoke_"):                        # the four tiles of __graft_entry__.smoke()
        k = int(name[6:])
        y, cb, cr = hevc_enc.synthetic_image(0xB200 + k, 128, 128, 8, True)
        return hevc_enc.encode_intra(y, cb, cr, log2_ctb_size=5, wpp=1, seed=0xB200 + k, **_vui())
    if name.startswith("bench_"):
        idx, log2ctb = (int(v) for v in name[6:].split("_ctb"))
        y, cb, cr = hevc_enc.synthetic_image(0xB200 + idx, 1024, 1024, 8, True)
        return hevc_enc.encode_intra(y, cb, cr, bit_depth=8, log2_ctb_size=log2ctb, qp=27, wpp=1, seed=0xB200 + idx, **_vui())
    return synth_stream(name)


HOST_NAMES = [c[0] for c in SYNTH + SYNTH_CPU_EXTRA] + [f"smoke_{k}" for k in range(4)] + [f"bench_{i}_ctb{l}" for i, l in BENCH_TILES]

# (w, h, chroma, log2ctb, qp, source, extra): cases of test_hevc_gpu_encoder.py's CONF and its QP-0 noise test
GPU_CASES = {
    "64x64-420-ctb32-qp0-synthetic": (64, 64, True, 5, 0, "synthetic", {}),
    "64x64-400-ctb64-qp37-noise": (64, 64, False, 6, 37, "noise", {}),
    "136x72-400-ctb32-qp51-synthetic": (136, 72, False, 5, 51, "synthetic", {}),
    "452x462-420-ctb32-qp37-synthetic-deblock": (452, 462, True, 5, 37, "synthetic", dict(beta_offset_div2=3, tc_offset_div2=-2)),
    "136x72-420-ctb32-qp22-noise-chroma_qp_offsets": (136, 72, True, 5, 22, "noise", dict(cb_qp_offset=4, cr_qp_offset=-3, slice_chroma_qp_offsets=1,
                                                                                          slice_cb_qp_offset=-2, slice_cr_qp_offset=2)),
    "1024x1024-400-ctb64-qp22-synthetic": (1024, 1024, False, 6, 22, "synthetic", {}),
    "256x128-420-ctb64-qp0-noise": (256, 128, True, 6, 0, "noise", {}),
}


def gpu_aus(enc, name):
    from test_hevc_gpu_encoder import source
    if name == "batch16-256x256-420-ctb32-qp27":        # the batch of test_deterministic_and_batch_independent
        return enc.encode([hevc_enc.synthetic_image(0xB200 + k, 256, 256, 8, True) for k in range(16)], qp=27)
    w, h, chroma, log2ctb, qp, kind, extra = GPU_CASES[name]
    return enc.encode([source(kind, w, h, chroma)], log2_ctb_size=log2ctb, qp=qp, **extra)


GPU_NAMES = list(GPU_CASES) + ["batch16-256x256-420-ctb32-qp27"]


def md5(aus):
    h = hashlib.md5()
    for au in aus:
        h.update(len(au).to_bytes(4, "big"))
        h.update(au)
    return h.hexdigest()


HOST_MD5 = {
    "ctb16_basic": "efa834709b825729f3733b07c59b25d7",
    "ctb16_nofilters": "3042d55866e365ce50e193a48390b61d",
    "ctb32": "b4eabb467541d5e43144f1f63443f28e",
    "ctb64": "fad18d4af994afa8d4dbc2bb9724349d",
    "ctb16_wpp_nosao": "31c9be54d1959646cbdfec9b5b2ca078",
    "ctb32_wpp_deep": "f030e2cd16e124bd05b578a07ec6a4ef",
    "ctb64_wpp_random": "d74c969c4f580fcc30f133e70c528b5a",
    "slices": "ad594fb582329ba46b84287628b1931a",
    "slices_nolf": "b964487df9a5ee83f6d34ff2cedcdeb2",
    "dependent_slices": "b4ce4891237187e1596d893f6b189a27",
    "slices_wpp": "916375bf53795d2382c3e815d000a162",
    "main10": "0c3f79ddce39b5c15147fd26dd84693b",
    "main12_wpp": "5a0caa57cee92628cde08661a8070dcc",
    "mono8": "96739c5aff407a3d53708d31ac8dd886",
    "mono10_ctb16_wpp": "8e064c839a5100234a2319d7dbd1dc04",
    "transform_skip": "60beb8f2a763c754f3779071a5ad1b5b",
    "chroma_qp_offsets": "5a6ee21bed0438543af88161b1f6ef64",
    "deblock_offsets": "4d770c622f8ef8da41763341270f79ea",
    "deblock_slice_override": "1491d0d80e746c26a1d740c35457a129",
    "deblock_slice_disabled": "1ce3831a187a3dc5c006518d7d86bfba",
    "odd_size_random": "7c9691ff4510f19395fea59768bd758b",
    "big_qp22": "048b25911e96009702718ed63632aa70",
    "big_qp37_vui": "5c83fd6f0f56aaae638297677deb9b82",
    "lowqp_deep": "1d3b8d8c204723d90de033be032be900",
    "highqp": "61f16e073448d993497510d000e067df",
    "tile_1024_like": "1746a3d7f8ebf43262a00c1e4f78c3cd",
    "scaling_default": "48e238510be9ba20331909f6318058a3",
    "scaling_sps_ctb64": "9be86f45bcd255e84d8d25977709881a",
    "scaling_pps_main10_tskip": "e6f2a279bf4bcdfb7c0b08b9cdb96326",
    "pcm": "be954aca6cb83309a04c2385c7e55b5b",
    "pcm_nolf_wpp_ctb64": "865a159237357390a4b9f75db1c17304",
    "pcm_nolf_main10": "acfcb33a68c6bae72694d2adb2efd287",
    "pcm_mono": "06e451eec9a93f6018d4dd13f104a60d",
    "bypass_mixed": "e8cd748bac085645de802655743d1a8e",
    "bypass_lossless": "95a0a72767a2ef2ff043589aea9d57a9",
    "bypass_tskip_main12": "81f56a17f08ea3c79f34fa933693010d",
    "pcm_bypass_scaling_slices_wpp": "ab79ee777919f8c2a169d7be4cfe08e7",
    "tiles_2x2": "6661785f8647df7cd951f8afda41a21c",
    "tiles_3x2_explicit_nolf": "d5d593e7d67307a1a0d726194f5dab26",
    "tiles_2x3_slice_per_tile_main10": "e7d1a335ec93c6644d7a8b908edd6c4d",
    "tiles_4x1_ctb64": "9dcf15771045d4ab620f9a597252e2b4",
    "tiles_5x4_ctb16_mono_nolf": "9f6ddd031a0f516d22af26665fc92447",
    "tiles_3x3_pcm_bypass_scaling": "75c9d3b9e693d3a81fdeb559c6c5c1f3",
    "x_main10_slices_wpp_tskip": "d5b2f7ea5c2b2cd582e1191145d98c7a",
    "x_ctb64_dependent_wpp": "68abf1119917c262d2b613283ec38012",
    "x_mono12_ctb64": "57ac9a6654a38d4072b4239d874ced44",
    "x_ctb16_deep_qp14": "c7c4fdb735178229ddd88ececf7d8cf3",
    "x_main12_highqp_nolf": "e1124009271e691cbb0bd79e9e5cb7a2",
    "x_odd_8bit_wpp_random": "19aaf5f73c01aa0b9c818e439eedf2b1",
    "x_main10_ctb64_qg8": "9f90e633b85bb818969b0888724122c9",
    "x_scaling_sps_mono_qp12": "2e9db289735a5c0438cb344cff625d1a",
    "x_scaling_pps_slices_wpp": "bd32f14ead880590b3d8eca0f3aba0c7",
    "x_bypass_mixed_nosao": "6c85389e9d0a0c2c1f3a8a1f94474a3a",
    "x_pcm_nolf_nosao_ctb16": "edc7bb4b4597c8f115dc85cf28877b91",
    "x_lossless_main10_ctb64_wpp": "8ff34f1c6c15b0a523d3e4dadbda1c58",
    "x_lossless_mono_nosao": "def54d6b85bd934320232581c52267fd",
    "x_tiles_2x2_main12_dqp_slice_per_tile": "4569e1332f404b2a56830927beb20a76",
    "x_tiles_1x3_slices_nolf_across_slices": "cf725bbf127be31e5956449958dcc445",
    "x_tiles_7x1_random_deep": "962aa23bd1d3c5bd189368214baa7ed9",
    "x_422_basic": "bfeafaabe0e30c6bc5bec70fbebef631",
    "x_444_basic": "bcd2cd5b45407b8be8e0d3b095a09506",
    "x_422_main10_random_tskip": "ddf2cba36ec7fc4bf3707c9d53f8410e",
    "x_444_main10_ctb16_random_tskip": "478980d5fbe38c9c8901038db71566d9",
    "x_422_main12_ctb64_deep_dqp": "c10da0344e9d9fd8550843d9ebf5dbf1",
    "x_444_ctb64_deep_dqp": "8eeb1249f8e3a86df3ebe9dfdaf1f7b3",
    "x_422_wpp_slices": "162a1e104213a3a35a3946901a302782",
    "x_444_wpp_slices": "7ac82118dd51dc6bfd168f20fd11007c",
    "x_422_pcm_bypass_nosao": "72d7195b76be992018c87201cf90ce85",
    "x_444_pcm_bypass_nosao": "fb33ef8d6723e192d4220891574290c6",
    "x_422_scaling_sps": "a88e6a919784af718e6bf6a7fd10c34b",
    "x_444_scaling_pps_ctb64": "5694374f0e2d4b7805f61ed7aa48e99f",
    "x_422_tiles_nolf": "544a12843fb6375518cf2bc4a94328a7",
    "x_444_lossless": "e021868f891d7a1abb820aac4ea0de7a",
    "x_422_lossless_main10": "e700e6bcb08168bea153c30405b9705f",
    "x_444_qp_offsets_pcm_nolf": "4f2d5841be3da41cd440959a0a5af862",
    "x_slices_every_row_nolf_across": "48ec665e6a70d2d0f1ddc74f2c7cabef",
    "smoke_0": "28692e4808b631b4b796356abfa36f39",
    "smoke_1": "8e0a799ca4d8f27228dc786982660545",
    "smoke_2": "6d0a71832328953c9f09d3c013b59dea",
    "smoke_3": "29b48bac070ae8e9a20f32c6f4ff2321",
    "bench_0_ctb5": "2b531e5f676d4355f881569077faea9d",
    "bench_3_ctb5": "867b0eeaceedde14a910e79269b2f25a",
    "bench_17_ctb5": "b30befd87f27eee4096b0e411673880d",
    "bench_0_ctb6": "3b55936f7edf656db26b27e37bf69d31",
    "bench_9_ctb6": "9e87050aaaed7fa512fab7745feb768e",
}

GPU_MD5 = {
    "64x64-420-ctb32-qp0-synthetic": "2be709ab571528c807f398b9489c780c",
    "64x64-400-ctb64-qp37-noise": "56c4c3a2eec1efcfc80a9598a0b160ad",
    "136x72-400-ctb32-qp51-synthetic": "ffc5f8702f09d2d41b3b66fdb2d5d3c5",
    "452x462-420-ctb32-qp37-synthetic-deblock": "8cd2efde9bb898ec0120b188b14c1b47",
    "136x72-420-ctb32-qp22-noise-chroma_qp_offsets": "c5ada01af69d81515d3090b6f08519df",
    "1024x1024-400-ctb64-qp22-synthetic": "4ffc619bcf188cc4d6c40a13713907b9",
    "256x128-420-ctb64-qp0-noise": "43afd4c1f9010c32d074230492e5c299",
    "batch16-256x256-420-ctb32-qp27": "f705cdad61babec984a9888ae90a53cb",
}


@pytest.mark.parametrize("name", HOST_NAMES)
def test_host_encoder_bytes(name):
    assert md5([host_au(name)]) == HOST_MD5[name]


@pytest.fixture(scope="module")
def gpu_enc(cuda):
    e = hevc_enc.GpuEncoder()
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_NAMES)
def test_gpu_encoder_bytes(gpu_enc, name):
    assert md5(gpu_aus(gpu_enc, name)) == GPU_MD5[name]
