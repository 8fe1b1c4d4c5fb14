"""CPU suite: libbftq.so loads and exports every symbol include/bftq.h declares.  No compute."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exports_match_header(built):
    hdr = open(os.path.join(ROOT, "include", "bftq.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(bftq_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 10
    lib = ctypes.CDLL(os.path.join(ROOT, "bftkv_b200", "libbftq.so"))
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, missing
    assert lib.bftq_version() == int(re.search(r"#define BFTQ_VERSION (\d+)", hdr).group(1))


def test_binding_loads_and_fails_loudly_without_gpu(built):
    import torch
    from bftkv_b200 import _lib, Engine
    _lib.load()
    if not torch.cuda.is_available():
        try:
            Engine(0)
        except _lib.BftqError as e:
            assert e.code == -1          # BFTQ_ERR_NO_DEVICE: no CPU fallback exists
        else:
            raise AssertionError("Engine() must fail without a CUDA device")


def test_sass_is_carry_free_imad_wide(built):
    """The radix-2^28 RSA kernel's inner loop must be plain IMAD.WIDE.U32 (no .X carry chain): that is
    the design of rsa_verify.cuh."""
    import subprocess
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    assert "sm_90a" in subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
    blocks = sass.split("Function :")
    rsa = [b for b in blocks if "rsa_verify_kernel" in b.split("\n")[0]]
    assert rsa
    for b in rsa:
        wide = len(re.findall(r"IMAD\.WIDE\.U32 ", b))
        widex = len(re.findall(r"IMAD\.WIDE\.U32\.X", b))
        assert wide > 100 and widex == 0, (wide, widex)


def test_sass_r32_kernel_resource_guard(built):
    """The radix-2^32 kernel every headline number comes from (rsa_verify_r32_kernel): carry-chained IMAD.WIDE.U32.X
    products, 128 registers (4 blocks x 128 threads per SM), at most a few spilled words, no local arrays, and the
    unified exponentiation loop: ONE general-product instance (4 owner steps x 2 x 57 chained multiplies = 456) plus
    ONE squaring instance of two owner steps (2 x 337) - the straight-line form carried five instances (2 326 wide
    multiplies, 7 440 instructions)."""
    import subprocess
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout
    name = "rsa_verify_r32_kernel"
    blk = [b for b in sass.split("Function :") if name in b.split("\n")[0]]
    assert len(blk) == 1, len(blk)
    widex = len(re.findall(r"IMAD\.WIDE\.U32\.X", blk[0]))
    instrs = len(re.findall(r"/\*[0-9a-f]{4,5}\*/\s+\S", blk[0]))
    assert 800 < widex < 1400 and instrs < 5600, (widex, instrs)
    m = re.search(r"Function [^\n]*" + name + r"[^\n]*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res)
    assert m
    regs, stack, shared, local = map(int, m.groups())
    assert regs <= 128 and stack <= 64 and local == 0 and shared <= 16384, (regs, stack, shared, local)
    assert widex == 456 + 2 * 337, widex       # mont_mul + mont_sqr x 2 owner steps


def test_sass_int_peak_loop_is_wide_multiplies_only(built):
    """bftq_measure_int_peak is the roofline denominator: its loop must issue the 64 carry-chained wide multiplies of
    eight steps and no other instruction on the multiplier pipe (an IMAD.MOV there makes the peak read low)."""
    import subprocess
    so = os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    blk = [b for b in sass.split("Function :") if "int_peak_kernel" in b.split("\n")[0]]
    assert len(blk) == 1
    ins = [(int(m.group(1), 16), m.group(2)) for m in re.finditer(r"/\*([0-9a-f]{4,5})\*/\s+([^;]+);", blk[0])]
    back = [(a, int(t, 16)) for a, op in ins for t in re.findall(r"BRA (?:`\()?0x([0-9a-f]+)", op) if int(t, 16) < a]
    assert len(back) == 1, back
    end, start = back[0]
    loop = [op.split()[0] if not op.startswith("@") else op.split()[1] for a, op in ins if start <= a <= end]
    wide = [o for o in loop if o.startswith("IMAD.WIDE")]
    other_imad = [o for o in loop if o.startswith("IMAD") and not o.startswith("IMAD.WIDE")]
    assert len(wide) == 64 and not other_imad, (len(wide), other_imad)
