"""GPU: tecogan_b200.jpeg.encode_jpeg writes the bytes cv2.imencode('.jpg') writes with its defaults, for every seeded
frame of tests/jpeg_cases.py (HR sizes up to 2160x3840, degenerate shapes, every residue of H and W modulo 16,
constant frames, constructed coefficient patterns), for a generator output, and through save_img in main.py --mode
inference (default extension) and test_while_train.  CV2_SHA256 records cv2's bytes for the seeded frames, so a frame
is checked against the live cv2 and against the recorded one (tests/test_jpeg_host.py checks the record on the host)."""
import argparse
import hashlib
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from tests import jpeg_cases as JC
from tests.conftest import GOLDEN, ROOT
from tests.test_gpu_png import _write_lr

CV2_SHA256 = {
    "constant": "6e1190e242581a6c4744dc11e8f7364f67a11523bb36e20096936c95a84b5223",
    "constant_1x1": "b75600195202cddab3ec8ea6dbcb5631282780d8c43dbee24d37a15df4f8d241",
    "constant_37x45": "85c2ff3da433c17da748fd9153c917157110d1a2a7e82e195b065d686e25f7fb",
    "extremes": "f1317297c161f89ee0ce4552d97910a64d76caae4fa9ebf43c4cc60c83ceba3a",
    "grid_15x1": "a89f7fd85cd3c08441025815edddca40335baeb1aae6b7bac9a9bf48d2a4ab4c",
    "grid_15x15": "27c4103ac9ccc9d8d1f45d4aaf7f90331d9720073a8606cbb4a3703deb50c4e1",
    "grid_15x16": "b2a695ea3749845c026275c8012035a0fbc87e1b1ac8964bd5c1245297f7f4ed",
    "grid_15x17": "19f8b2a08a113f725e41fffabbfa236bdc3961a29507661494d2ae032dde2190",
    "grid_15x24": "7df485777aa3522408881f2964ca1dedcbd495788ec9cbfd1ab747aa0fd705cc",
    "grid_15x33": "1689126b36a3b006b49a244bb1c390750d910a58803a5e09699da6b89abcd760",
    "grid_15x7": "e2a8c382a98f43f5da1f78419d94b2a75828cbb25350a779b19a6aad405be5a1",
    "grid_15x8": "7011e8b5dbc65f8eb6244e0e42b924e6f1c08744f5ae191ebb073df0c34885e7",
    "grid_15x9": "e799ccd4b3f1770d689670d0fea85a6e275a1358c86c9c173474224a3e108426",
    "grid_16x1": "ccdd182409d67cb6fd6d6798067e8b8a0c6f1885d6d2ed10bec82e9aef2ec052",
    "grid_16x15": "7e228a840a6d782ad87b14ace6ac351fb52c85f03a99c98fdb0fd8c144927434",
    "grid_16x16": "78b01c5e37b33fad2ebd0cce712dc697ae4116b9b2eca39557edc06a262ce2b9",
    "grid_16x17": "7d0eeded8248dc4d9d008d3cb162e923460c6afa4975db610aedaa6280a736b9",
    "grid_16x24": "3f87cac1cfe42b1dd9f1eccec051b5d03f51047f4e76e9fda2cc02fdbc00ae58",
    "grid_16x33": "46fc417f8ca1600ea94be400c92bd81ef5f986c2d79b4baf9ecac2449ba23705",
    "grid_16x7": "1ad19aa5234379ab38e8825cbb6101a0e1662530343291aa652b85a21cb77ad9",
    "grid_16x8": "252decc6725bedddc830f9c87b60a90b3e93d51f4c8f2e71d1841aa67839f891",
    "grid_16x9": "cd061164d8ce627ec700f8cedf59a5a150884fcca627f0bd9a08b88c9a7c1c88",
    "grid_17x1": "64ff7cbeb4b00cdaeae0daa7d58a3242a461080802d20dd6f85bd9e3c12a3e6b",
    "grid_17x15": "c58ccde76e07699d4545b6fecb9f6e59c5f6661ceb470603ac506daeece6a0d1",
    "grid_17x16": "0cf496d638287c1a206809e8f8afff01102af449e802a63c791a774efac68bc7",
    "grid_17x17": "21ae99ffc767f29371305fa8269fed3316e368f8309ffb8e2c2a6e0cc0cfea4b",
    "grid_17x24": "abd767a15b4d7879e138b53115e532d2532b72e81969225d89b33eb739b99b06",
    "grid_17x33": "d80dfef1c9796c1bbff68b93a07353d7db0c9b01ef2c8fec9fa400238a810b2e",
    "grid_17x7": "f9c5f022d3c065b382a6a5297e0b3e2387b86a2e16fc272df76a30a91dab7a03",
    "grid_17x8": "2dc5de3186fcf274caf35a6a16c62a45a3b44550fa4b281fa552a658bd82fe99",
    "grid_17x9": "4042afe490efa1e5416971d21e5bb334f3bc1027b4286eb2d488cde89837dddb",
    "grid_1x1": "f6d45a55e4896a96d44699e1bf5dc6bbc6c1ca9261bbe98f5423184d02aa75b8",
    "grid_1x15": "8afe6e0443133111ba4749f71e1484014f772e8ad896c88079773598f065b425",
    "grid_1x16": "50df7615fd60751dcbc6fe50bf3420aa470496396e993d0a47bc08c0e3e34ae8",
    "grid_1x17": "ecc6354418645e7df27eb8158319c1fe1c1d1c999d28a7fc6d4d679550b716b1",
    "grid_1x24": "1f7a97c6133f1bcb9ac52cfd6d1f5d25fcafb842d4184d7cfb75177198b9da98",
    "grid_1x33": "0e01852854fe16738aab80c539b235492ff48551e392e114d41e3c5c64808e57",
    "grid_1x7": "36954dc51dd23e772f5577ae1be651fe92593e6b8567a28e705f5a740897c8d7",
    "grid_1x8": "a45ef05047be04990133ccabd778842aeb4dfc3a24f7c56e6fca98c5e40828ad",
    "grid_1x9": "ccc9486325442115dd956def296b484d89d44dcd971fcfc95a0e2a9725a0ee81",
    "grid_24x1": "dd8a50a55673f5f153bd28d68238e85688b6ae1bb79ba2695bcfa3d9ee337882",
    "grid_24x15": "24d94bb49b467855f10abedbe74e5f7732e1829dfacdffbf3b9dec0e81a73d57",
    "grid_24x16": "67eb3dc68e2d8d052551b26a74760a441a980bc1dd370bd5ff70f58d3d643edc",
    "grid_24x17": "a5ef944ab1dd4c58b89c1c2e807f87215c59bb38483665b79558ac1ec415db3b",
    "grid_24x24": "2287b2e3b7b185a7bf235735587d69e369f90bf646fa91b1cf56d811fd8e7270",
    "grid_24x33": "30829a0adad6842450bec36c62351923a6bd44f7cc88079f721f6c6fd5bad3ff",
    "grid_24x7": "ba84755acc0e5e3b2a1e4f26a8bc63cd50e148f7df61c3e62ca899f8b8484fec",
    "grid_24x8": "02bbe0a801ac069b43a0e63cd20ea477e60a64faeac93d22a08975c63dee3027",
    "grid_24x9": "7dbfd9c4c056f8d623240afe254b6f56a7ea154d2b75745a29f7bc57bd1d84db",
    "grid_33x1": "564198cefb9960a837bc0a77f19675f1002aa01b0462d492665eea5a0499f432",
    "grid_33x15": "815bce09150192b68657bb79a93cba9596c71d12b1b3360a4266213335fb3804",
    "grid_33x16": "62f4235c08b0d6c37f0409bed309bc9f9513c97ad9d34732406296567d1a554e",
    "grid_33x17": "b23104063810affd6487a38a1ac00333d1ea087548b95b5e74aadc7e2babc3af",
    "grid_33x24": "cac9a9515dc3f2918d5b57100b674cf9ab76367268d06e199048bede1887a8c9",
    "grid_33x33": "52a4fc34d731db3fc19ebbdd53eab0f9c15e4b90ba105639e38a4e90ad5850fd",
    "grid_33x7": "61b50ebbf98c2e8d51e1b2830750ef1ddabe9c33380f4c85104a07687e70d351",
    "grid_33x8": "91c27b5e6bfe20bc4d5ec86d5bac7d6f6210eaae7b125b8039243d3eebfb0b11",
    "grid_33x9": "1231eb5c290717d152ab02495c319b5bca541e195b3d731dda4d91dab0a9c765",
    "grid_7x1": "7ea047871265f997ef8b923cde1b3cf1510200a61732f9d1e6070bcb325a3649",
    "grid_7x15": "341626bd5d4c8fc931a6fa6babbe70c586e64cb45e7d5f807953a71f06cec824",
    "grid_7x16": "0cb961ca3c3bf513537b583ee26069ce91e3998c2d8a5da048dd21612cbc61df",
    "grid_7x17": "69617fa22a23678d2812b1afa3f76384b96b4ad14f4ac25dbff8e60c5d8d5da6",
    "grid_7x24": "46ff40a536fee0bb5a826e4556a2d3b79dbb6c7cdef0a935573e87c716a5b38f",
    "grid_7x33": "d52f5dcc89d69ebcc2659c6fd655502b6dba2a4d3628f0b73eb24bc84e0a8e67",
    "grid_7x7": "8cd5226fb3baca2a422cc6fa313b83f19dc75073329eba70a167a08e34d90058",
    "grid_7x8": "aeedb1239d8b002dca2be3776a98558d3f9f71c21cdf26666b01200ce2d9eb9d",
    "grid_7x9": "ef14e5ecee8b17bd242a61051abf716f97c6b3aa6e632c6ea1ef58dd6799f738",
    "grid_8x1": "94ebc3124e5685f2b68baa163f270438fc3818ed43b015250e570fe73c44d083",
    "grid_8x15": "71ed477d99d5bef9e28831d5df8bba50c4179f562c4b3c66ef4745a2e858459c",
    "grid_8x16": "d1550d603fee9547dd5256460734448c1d5f4df40e6c8c2cb6bee00c87c0425d",
    "grid_8x17": "96fe52b3c6ef2eaf53ceec74821dbf88162230579b0157e5eb81b7eb0f59c97c",
    "grid_8x24": "5a2953e71277f73f95ab532cb5b7d4938366121ed89e93a4cb1df896e59ea651",
    "grid_8x33": "33d6fb9d5d27cc5322a0d737d4d41991852d503551e32321e6b45a407dc2d69f",
    "grid_8x7": "f3432d7016552fee9837049ffa0b18becd615740b570405b2841a13b09f99769",
    "grid_8x8": "fe5b84331d8ab5b3e29b2c02f84bbef814f27b48813cfaeee321fb1577caa430",
    "grid_8x9": "1098ab3d1eefd3b676a46016983dc4eaac3ab0b71a3dcc5e340a8e315ca3019f",
    "grid_9x1": "4768175913be9c853feab9c5ae9c154d6c3f2d688cf6100f0d671dcabd6f2bb9",
    "grid_9x15": "d9d6f5f20f16e4f271f339210ed39b0d99a9de5a1e13fcce5d90e9a4e499d4a8",
    "grid_9x16": "6dc335d71768833ab1192434413c2d8143d21d0f5bf1fd1ebcdfb9af5930c60e",
    "grid_9x17": "dd5e8faabb62377d5e3049544297a9a5ff5e8fef0f2992d1e18160a833ff8efe",
    "grid_9x24": "5ccba36d67eade57e8445ac5f9e2806da8e51d3b51bbc2b0faf9c3e7d62f4ab7",
    "grid_9x33": "5dd0b956f40ca37afdfb3aac3fe8d5823b389b6b869b881eb3e5c403b346d23a",
    "grid_9x7": "14ead093afae22534a9e26847e5b035fd02adb4e087cf9ea0807ef59cba7e824",
    "grid_9x8": "f6a9e1ac4de12e5957092026335d08771d0823d3ceef4579f704665622d59c95",
    "grid_9x9": "1e5356210b9bd3ec076882f73250364da117f94110dd9133968b46d636bdaf56",
    "noise_1x1": "3e86344bf2a08b17c78bfc10365666eb43e257b9187099e5ae5788a16ab0e52f",
    "noise_1x257": "a93159d67642ba55849bdd39f6d5225ea053461a4f26319af1567912bdafad6d",
    "noise_300x1": "e08ff21da44313e62be1aa23d428b3255df2c5095275112e6be1b98f189439c1",
    "noise_576x720": "6ff5bdd0ffd0a44c8a2d88e526cb299c59e031c36765f9edfc92c8a289236137",
    "runs": "d9088a74b9ad7286e5f03f1b38035c1bf7c6bf4794d115a72018ef4f8f16f9d9",
    "smooth_1080x1920": "d83df0e96d19381932fd560d3dc3b6677ddfc36fc629f5ac1f7b507a4ea39c88",
    "smooth_128x128": "9dddfcd8f44fbd3e8ef788f64a19d31099ed2bfe9f2b1367bd1cad206269f457",
    "smooth_2160x3840": "bebcccf4c4a70f53b9c85e9285471167e88a7f23533931ccc9f25295e56792ec",
    "smooth_32x32": "c453e91d3ff093c3a4806bc40330c1bdc708349e2be97bc8549b253587f40b86",
    "smooth_576x720": "8dacdfc748cfc144e126684518507575229bf6745504e8313df2cd1e372e7c88",
    "smooth_99x201": "0024ea355ff44869a18ce642253ffa5e2a0a956d782abf2a5728a697260326cb",
}


def _cv2_jpg(rgb):
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(rgb[:, :, ::-1]))
    assert ok
    return buf.tobytes()


@pytest.fixture(scope="module")
def cases():
    return JC.cases()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CV2_SHA256))
def test_encode_matches_cv2(cases, name):
    from tecogan_b200.jpeg import encode_jpeg
    rgb = cases[name]
    got = encode_jpeg(torch.from_numpy(rgb).cuda())
    ref = _cv2_jpg(rgb)
    assert hashlib.sha256(ref).hexdigest() == CV2_SHA256[name]
    assert got == ref, (name, len(got), len(ref))


@pytest.mark.gpu
def test_repeated_calls_reuse_buffers(cases):
    from tecogan_b200 import jpeg
    a, b = cases["smooth_128x128"], cases["smooth_99x201"]
    first = jpeg.encode_jpeg(torch.from_numpy(a).cuda())
    ws = jpeg._state["ws"].data_ptr()
    for _ in range(3):
        assert jpeg.encode_jpeg(torch.from_numpy(a).cuda()) == first
    assert jpeg._state["ws"].data_ptr() == ws
    assert jpeg.encode_jpeg(torch.from_numpy(b).cuda()) == _cv2_jpg(b)      # another size, then back
    assert jpeg.encode_jpeg(torch.from_numpy(a).cuda()) == first


@pytest.mark.gpu
def test_rejects_bad_input():
    from tecogan_b200.jpeg import encode_jpeg
    with pytest.raises(ValueError):
        encode_jpeg(torch.zeros(4, 4, 3, dtype=torch.uint8))                  # CPU tensor
    with pytest.raises(ValueError):
        encode_jpeg(torch.zeros(4, 4, 3, device="cuda"))                       # float
    with pytest.raises(ValueError):
        encode_jpeg(torch.zeros(4, 4, 4, dtype=torch.uint8, device="cuda"))   # not RGB
    with pytest.raises(ValueError):
        encode_jpeg(torch.zeros(4, 6, 3, dtype=torch.uint8, device="cuda")[:, ::2])
    with pytest.raises(ValueError):
        encode_jpeg(torch.zeros(0, 4, 3, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        encode_jpeg(torch.zeros(1, 65501, 3, dtype=torch.uint8, device="cuda"))


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments():
    from tecogan_b200 import _ffi, jpeg
    ws, cap = jpeg.plan_bytes(16, 16)
    x = torch.zeros(16, 16, 3, dtype=torch.uint8, device="cuda")
    w = torch.empty(ws, dtype=torch.uint8, device="cuda")
    o = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = torch.empty(1, dtype=torch.int64, device="cuda")
    f = _ffi.lib().teco_jpeg_encode_rgb8
    s = _ffi.stream_ptr()
    assert f(_ffi.ptr(x), 16, 16, _ffi.ptr(w), ws - 1, _ffi.ptr(o), cap, _ffi.ptr(n), s) == -1
    assert f(_ffi.ptr(x), 16, 16, _ffi.ptr(w), ws, _ffi.ptr(o), cap - 1, _ffi.ptr(n), s) == -1
    assert f(None, 16, 16, _ffi.ptr(w), ws, _ffi.ptr(o), cap, _ffi.ptr(n), s) == -1
    assert f(_ffi.ptr(x), 16, 16, None, ws, _ffi.ptr(o), cap, _ffi.ptr(n), s) == -1
    assert f(_ffi.ptr(x), 16, 16, _ffi.ptr(w), ws, None, cap, _ffi.ptr(n), s) == -1
    assert f(_ffi.ptr(x), 16, 16, _ffi.ptr(w), ws, _ffi.ptr(o), cap, None, s) == -1
    assert f(_ffi.ptr(x), 0, 16, _ffi.ptr(w), ws, _ffi.ptr(o), cap, _ffi.ptr(n), s) == -1
    assert f(_ffi.ptr(x), 16, 0, _ffi.ptr(w), ws, _ffi.ptr(o), cap, _ffi.ptr(n), s) == -1
    for h, wd in ((16, 0), (0, 16), (65501, 16), (16, 65501)):
        with pytest.raises(ValueError):
            jpeg.plan_bytes(h, wd)
    assert jpeg.plan_bytes(65500, 1)[0] > 0


@pytest.mark.gpu
def test_generator_output_576x720():
    """The calendar fixture through the generator with seeded weights: an HR frame as save_img quantises it."""
    from oracle import teco_oracle as O
    from tecogan_b200 import config, kernels as K, variables as V
    from tecogan_b200.engine import InferenceEngine
    from tecogan_b200.jpeg import encode_jpeg
    pg, pf = O.damp_generator(O.init_generator(seed=1234, num_resblock=4)), O.init_fnet(seed=4321)
    V.set_default_store(V.VariableStore()).load({**pg, **pf})
    config.set_precision("fp32")
    fr = np.load(os.path.join(GOLDEN, "calendar_lr.npz"))["full_u8"][:3].astype(np.float32) / 255.0
    outs = InferenceEngine(144, 180, 4).run_sequence([torch.from_numpy(f).cuda() for f in fr])
    for o in outs:
        u8 = K.to_u8(o[0]).contiguous()
        assert tuple(u8.shape) == (576, 720, 3)
        assert encode_jpeg(u8) == _cv2_jpg(u8.cpu().numpy())


def _same_as_lossless(jpg_dir, bmp_dir, names):
    """Every .jpg equals cv2's JPEG of the frame the host path wrote losslessly as .bmp."""
    assert names
    for name in names:
        rgb = cv2.imread(os.path.join(bmp_dir, name + ".bmp"), cv2.IMREAD_UNCHANGED)[:, :, ::-1]
        got = open(os.path.join(jpg_dir, name + ".jpg"), "rb").read()
        assert got == _cv2_jpg(rgb), name


@pytest.mark.gpu
def test_main_inference_default_jpg_end_to_end(tmp_path):
    """main.py --mode inference with no --output_ext writes .jpg files, byte-identical to cv2's."""
    _write_lr(str(tmp_path))
    for ext in (None, "bmp"):
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
            os.path.join(ROOT, "main.py"), "--mode", "inference", "--checkpoint", "random:5", "--num_resblock", "2",
            "--input_dir_LR", "./LR/calendar/", "--output_dir", "out_" + (ext or "default"), "--output_pre", "",
            "--cudaID", os.environ.get("CUDA_VISIBLE_DEVICES", "0")] + (["--output_ext", ext] if ext else [])
        r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    files = sorted(os.listdir(str(tmp_path / "out_default")))
    assert len(files) == 8 and all(f.endswith(".jpg") for f in files), files
    _same_as_lossless(str(tmp_path / "out_default"), str(tmp_path / "out_bmp"), [f[:-4] for f in files])


@pytest.mark.gpu
def test_while_train_jpg(tmp_path, monkeypatch):
    import main as M
    from oracle import teco_oracle as O
    from tecogan_b200 import variables as V
    _write_lr(str(tmp_path), n=10)
    monkeypatch.chdir(str(tmp_path))
    pg, pf = O.damp_generator(O.init_generator(seed=7, num_resblock=2)), O.init_fnet(seed=8)
    V.set_default_store(V.VariableStore()).load({**pg, **pf})
    for ext in ("jpg", "bmp"):
        fl = argparse.Namespace(output_dir=str(tmp_path / ("run_" + ext)), precision="fp32", num_resblock=2,
                                output_ext=ext)
        M.test_while_train(fl, 3)
    names = ["000000003_%04d" % i for i in range(1, 11)]
    assert sorted(os.path.splitext(f)[0] for f in os.listdir(str(tmp_path / "run_jpg" / "train"))) == names
    _same_as_lossless(str(tmp_path / "run_jpg" / "train"), str(tmp_path / "run_bmp" / "train"), names)


# The extensions cv2 4.13 writes as JPEG, all with the same bytes; it rejects .jfif.
JPEG_EXTS = (".jpg", ".jpeg", ".jpe")


@pytest.mark.gpu
def test_save_img_routes_and_unwritable_path(cases, tmp_path, monkeypatch):
    """.JPG, .jpeg and .jpe go to the device encoder, with cv2's bytes; an unwritable path is ignored as cv2.imwrite's
    False is; a numpy image still goes to cv2.imwrite."""
    from tecogan_b200 import jpeg
    from tecogan_b200.lib import ops
    from tecogan_b200 import kernels as K
    img = torch.from_numpy(cases["smooth_99x201"]).cuda().float() / 255.0
    rgb = K.to_u8(img).cpu().numpy()                              # the frame save_img quantises
    bgr = np.ascontiguousarray(rgb[:, :, ::-1])
    ref = _cv2_jpg(rgb)
    for ext in JPEG_EXTS:
        ok, buf = cv2.imencode(ext, bgr)
        assert ok and buf.tobytes() == ref, ext
    with pytest.raises(cv2.error):
        cv2.imencode(".jfif", bgr)
    calls = []
    real = jpeg.encode_jpeg
    monkeypatch.setattr(jpeg, "encode_jpeg", lambda t: calls.append(t.shape) or real(t))
    for name in ("a.JPG", "b.jpeg", "c.jpe"):
        ops.save_img(str(tmp_path / name), img)
        assert open(str(tmp_path / name), "rb").read() == ref, name
    assert len(calls) == 3
    ops.save_img(str(tmp_path / "missing" / "d.jpg"), img)
    assert len(calls) == 4 and not os.path.exists(str(tmp_path / "missing"))
    ops.save_img(str(tmp_path / "e.jpg"), rgb.astype(np.float32) / 255.0)
    assert len(calls) == 4 and os.path.getsize(str(tmp_path / "e.jpg")) > 0
