"""Registers, stack bytes and the Forward / Backward column loops of every k_posterior_sm instantiation.

Usage: python tests/sass_cells.py [library]   (default: muscle_b200/libmuscle_b200.so)

The plain-mode passes compute two rows per lane per step and the MEGA-mode passes one, so a column loop
computes R = 2 or 1 cells per iteration.  A column loop is the innermost backward branch whose body holds
8*R FFMA.RP (8 per LOG_ADD of each cell); the first in the code is the Forward loop, the second the Backward
loop (any other number of such loops is reported with a warning and the loops are listed in code order).
For each it prints R, the loop's length in instructions, the FADD / FFMA.RP / LDS.128 / STS.128 / LDG counts
per iteration, and the length per cell, the figure to compare across R.  Not a test: it reads the
compiler's output, and the counts are what a change to the kernel is checked against.
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);")
KERNEL = re.compile(r"_Z14k_posterior_smILb(\d)ELi(\d+)ELb(\d)EEv10PostParams")
COUNTED = ("FADD", "FFMA.RP", "LDS.128", "STS.128", "LDG")


def counted(op):
	base = op.split(".")[0]
	return {"FADD": base == "FADD", "FFMA.RP": op == "FFMA.RP", "LDS.128": base == "LDS" and op.endswith(".128"),
	  "STS.128": base == "STS" and op.endswith(".128"), "LDG": base == "LDG"}


def column_loops(insns):
	"""[(start, end, R)]: the innermost backward branches with 8*R FFMA.RP in their body, R = 1 or 2"""
	addr = {a: k for k, (a, _, _) in enumerate(insns)}
	loops = []
	for k, (a, op, args) in enumerate(insns):
		t = re.match(r"(?:P\d,\s*)?0x([0-9a-f]+)", args)
		if op.startswith("BRA") and t and int(t.group(1), 16) < a and int(t.group(1), 16) in addr:
			s = addr[int(t.group(1), 16)]
			n = sum(op2 == "FFMA.RP" for _, op2, _ in insns[s:k + 1])
			if n in (8, 16):
				loops.append((s, k, n//8))
	return [(s, e, r) for s, e, r in loops if not any(s <= s2 and e2 <= e and (s2, e2) != (s, e) for s2, e2, _ in loops)]


def main():
	lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "muscle_b200", "libmuscle_b200.so")
	out = subprocess.run(["cuobjdump", "-sass", "-res-usage", lib], check=True, capture_output=True, text=True).stdout
	res = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+)", out))
	for body in out.split("Function : ")[1:]:
		name = body.split(None, 1)[0]
		m = KERNEL.fullmatch(name)
		if not m:
			continue
		insns = [(int(a, 16), op, args) for a, _, op, args in INSN.findall(body)]
		print("%s CM=%-2s %s  %s" % ("MEGA " if m.group(1) == "1" else "plain", m.group(2),
		  "DUMP" if m.group(3) == "1" else "prod", res.get(name, "?")))
		loops = column_loops(insns)
		if len(loops) != 2:
			print("    warning: %d column loops found, expected Forward and Backward; listed in code order" % len(loops))
		labels = ("Forward ", "Backward") if len(loops) == 2 else ["loop %-3d" % k for k in range(len(loops))]
		for label, (s, e, r) in zip(labels, loops):
			n = {c: sum(counted(op)[c] for _, op, _ in insns[s:e + 1]) for c in COUNTED}
			print("    %s R=%d %3d  %s  | per cell %.1f" % (label, r, e - s + 1, "  ".join("%s %d" % kv for kv in n.items()),
			  (e - s + 1)/r))


if __name__ == "__main__":
	main()
