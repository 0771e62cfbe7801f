"""Code-generation guards for the 2^11-point NTT pass rounds, which are bound by the integer ALU pipe (DESIGN §9): the shared-memory
accesses of a round are a row pointer plus a compile-time offset, the forward write-back is unrolled over its rows the same way, the
butterfly's sum is folded on the FMA pipe, and the shifts by 2^64 .. 2^95 multiply with one IMAD.WIDE. Needs no GPU: the objects build() compiled, and two one-line kernels compiled here, are
disassembled."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "winterfell_b200", "_build")
CSRC = os.path.join(ROOT, "winterfell_b200", "csrc")
CUDA_BIN = "/usr/local/cuda/bin"
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(CUDA_BIN, "cuobjdump")
NVCC = shutil.which("nvcc") or os.path.join(CUDA_BIN, "nvcc")

# Hopper's integer ALU pipe: adds, logic, shifts, selects, compares. IMAD* (including IMAD.X / IMAD.WIDE) issue to the FMA pipe.
ALU = ("IADD3", "LOP3", "SHF", "SEL", "ISETP", "LEA", "PLOP3")


def _sass(path):
    out = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True, check=True).stdout
    fns, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            fns[cur] = []
        elif cur and re.match(r"\s+/\*[0-9a-f]{4,6}\*/", line):
            fns[cur].append(line.strip().split("/* 0x")[0].strip())  # "/*addr*/ [predicate] OPCODE operands ;"
    return fns


def _op(ins):
    return re.sub(r"^@!?U?P[0-9T]\s+", "", re.sub(r"^/\*[0-9a-f]+\*/\s+", "", ins)).split()[0].rstrip(";")


@pytest.mark.skipif(not (os.path.exists(os.path.join(BUILD, "ntt2.o")) and os.path.exists(CUOBJDUMP)),
                    reason="objects not built (python -c 'import __graft_entry__ as g; g.build()') or no cuobjdump")
def test_round_accesses_and_alu_work():
    fns = _sass(os.path.join(BUILD, "ntt2.o"))
    big = {n: l for n, l in fns.items() if "ntt2_pass_kernel" in n and "Li11E" in n}
    assert len(big) == 2, list(fns)
    for name, lines in big.items():
        smem = [i for i in lines if _op(i).startswith(("LDS", "STS"))]
        imm = [i for i in smem if re.search(r"\[R\d+(\+UR\d+)?\+0x[0-9a-f]+\]", i)]
        # 3 rounds x 32 accesses in the task bodies (91 of 119 shared accesses at this writing); the form that computed every row
        # index (XOR, shift, lane insert, scale: four instructions per access) had 23 of 119
        assert len(imm) >= 64 and len(imm) >= 0.6 * len(smem), (name, len(imm), len(smem))
        # ALU-pipe instructions of the three round loops (a task body each: shared loads and stores, 400-2000 instructions,
        # closed by a backward branch): 1529-1530 at this writing, 1762-1763 before the row pointers, the folded butterfly
        # sum and the one-IMAD.WIDE high shifts
        addr = [int(re.match(r"/\*([0-9a-f]+)\*/", i).group(1), 16) for i in lines]
        ops = [_op(i) for i in lines]
        rounds = []
        for a, o, i in zip(addr, ops, lines):
            m = re.search(r"BRA\S*\s+(?:U?!?P\d,\s+)?(?:`\()?.*?0x([0-9a-f]+)", i)
            if o.startswith("BRA") and m and int(m.group(1), 16) < a:
                body = [oo for aa, oo in zip(addr, ops) if int(m.group(1), 16) <= aa <= a]
                if 400 < len(body) < 2000 and any(x.startswith("LDS") for x in body) and any(x.startswith("STS") for x in body):
                    rounds.append(sum(x.startswith(ALU) for x in body))
        assert len(rounds) == 3 and sum(rounds) <= 1600, (name, rounds)
        # the forward write-back: sixteen 128-bit row stores from row pointers, besides the generic loop's four
        assert sum(o.startswith("STG.E.128") for o in ops) >= 20, name


def _one_kernel(tmp_path, body):
    src = tmp_path / "k.cu"
    src.write_text('#include "gl64.cuh"\n__global__ void k(u64* v) {\n    const u32 i = threadIdx.x;\n' + body + "\n}\n")
    cubin = tmp_path / "k.cubin"
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + CSRC, "-cubin", str(src), "-o", str(cubin)],
                   check=True, capture_output=True)
    (lines,) = _sass(str(cubin)).values()
    # the arithmetic only: drop the loads, stores, control and the address computation (index x 8) around it
    return [_op(i) for i in lines if not _op(i).startswith(("LDG", "STG", "S2R", "S2UR", "ULDC", "LDC", "EXIT", "BRA", "NOP"))
            and not re.search(r", 0x8,", i)]


@pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)), reason="no nvcc / cuobjdump")
def test_butterfly_pipe_split(tmp_path):
    ops = _one_kernel(tmp_path, "    u64 a = v[i], b = v[i + 1024];\n    gl_butterfly(a, b);\n    v[i] = a;\n    v[i + 1024] = b;")
    alu = sum(o.startswith(ALU) for o in ops)
    fma = sum(o.startswith("IMAD") for o in ops)
    # sum: 64-bit add, carry test, one IMAD.WIDE fold; difference: borrow chain. With the a - (p - b) sum it was 11 ALU + 2 FMA.
    assert alu <= 9 and fma <= 4 and any(o.startswith("IMAD.WIDE") for o in ops), ops


@pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)), reason="no nvcc / cuobjdump")
@pytest.mark.parametrize("k", [72, 84])
def test_high_shift_has_no_imad_hi(tmp_path, k):
    ops = _one_kernel(tmp_path, f"    v[i] = gl_mul_2exp<{k}>(v[i]);")
    assert not any(o.startswith("IMAD.HI") for o in ops) and any(o.startswith("IMAD.WIDE") for o in ops), ops
