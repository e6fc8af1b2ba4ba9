// Host-only harness: the engine's own mix64 (csrc/apo_device.cuh, __host__ __device__) and the corpus digest's home slot
// (csrc/apo_kernels.cu cd_insert) over keys read from stdin, so that tests/flagship_fixtures.py's Python restatement can be
// compared with them.  Input: n, nslots, then n x {d2 bits, slots} (uint64, native order).  Output: n x {mix64(d2 bits),
// home slot}.  Built with nvcc, run on the CPU.
#include <cstdio>
#include <vector>
#include "apo_device.cuh"

int main() {
	unsigned long long n = 0, nslots = 0;
	if (fread(&n, 8, 1, stdin) != 1 || fread(&nslots, 8, 1, stdin) != 1) return 2;
	std::vector<unsigned long long> in(2 * n), out(2 * n);
	if (fread(in.data(), 8, 2 * n, stdin) != 2 * n) return 2;
	for (unsigned long long i = 0; i < n; i++) {
		const unsigned long long x = in[2 * i], y = in[2 * i + 1];
		out[2 * i] = apo::mix64(x);
		out[2 * i + 1] = apo::mix64(x ^ apo::mix64(y + apo::GOLD)) & (nslots - 1);
	}
	fwrite(out.data(), 8, 2 * n, stdout);
	return 0;
}
