"""Device selection lives in one place: b2::DeviceScope (b2_internal.hpp, b2_context.cu) is the only code in the library that calls
cudaSetDevice.  Entry points open the scope instead (B2_ON_DEVICE), and it hands the caller's current context back on return; a
cudaSetDevice anywhere else would leave the caller on the library's device."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gtsam_points_b200", "csrc")


def _code(path):
    """The source with comments and string literals blanked out (line breaks kept, so line numbers still hold)."""
    src = open(path).read()
    return re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"', lambda m: re.sub(r"[^\n]", " ", m.group()), src, flags=re.S)


def test_only_the_device_scope_selects_a_device():
    outside, inside = [], 0
    for name in sorted(os.listdir(CSRC)):
        code = _code(os.path.join(CSRC, name))
        scope = re.search(r"^DeviceScope::DeviceScope\(int device\) \{.*?^\}", code, flags=re.S | re.M)  # the scope's constructor
        for m in re.finditer(r"\bcudaSetDevice\b", code):
            if scope and scope.start() <= m.start() < scope.end():
                inside += 1
            else:
                outside.append(f"{name}:{code.count(chr(10), 0, m.start()) + 1}")
    assert not outside, "cudaSetDevice outside b2::DeviceScope (open the scope with B2_ON_DEVICE instead): " + ", ".join(outside)
    assert inside == 1
