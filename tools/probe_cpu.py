"""Host probe: CPU model, thread count and the accuracy of torch's CPU fp32 matmul."""
import os, torch
print("cpu_count", os.cpu_count(), "torch threads", torch.get_num_threads())
try:
    print([l for l in open("/proc/cpuinfo") if "model name" in l][0].strip())
    print([l for l in open("/proc/cpuinfo") if l.startswith("flags")][0][:2000].count("amx"), "amx flags")
except Exception as e:
    print(e)
g = torch.Generator().manual_seed(0)
for (m, k, n) in [(48, 512, 48), (256, 2048, 256), (200, 256, 5000)]:
    a, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g)
    err = ((a @ b.t()).double() - a.double() @ b.double().t()).abs().max().item()
    print(f"fp32 matmul {m}x{k}x{n}: max abs err vs fp64 {err:.3e}")
print(torch.__config__.show()[:600])
