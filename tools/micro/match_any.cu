// microbenchmark: latency of __match_any_sync / ballot / shfl / smem atomics on sm_90a
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(unsigned *out, long long *cyc, int mode)
{
	__shared__ unsigned tab[4096];
	unsigned lane = threadIdx.x;
	unsigned v = (mode & 1) ? lane * 2654435761u : 7u;       // distinct or identical values
	for (int i = lane; i < 4096; i += 32) tab[i] = 0;
	__syncwarp();
	unsigned acc = 0;
	long long t0 = clock64();
	for (int i = 0; i < 1000; i++) {
		unsigned x = v + acc;                                // dependent chain
		if (mode < 2) acc += __match_any_sync(0xffffffffu, x);
		else if (mode == 2) acc += __ballot_sync(0xffffffffu, x & 1);
		else if (mode == 3) acc += __shfl_sync(0xffffffffu, x, (lane + 1) & 31);
		else if (mode == 4) acc += atomicOr(&tab[(x >> 8) & 4095], 1u << (x & 31));
		else if (mode == 5) { tab[(x >> 8) & 4095] = x; __syncwarp(); acc += tab[((x >> 8) + 1) & 4095]; }
		else if (mode == 6) acc += __reduce_add_sync(0xffffffffu, x);
	}
	long long t1 = clock64();
	out[lane] = acc;
	if (lane == 0) cyc[0] = (t1 - t0) / 1000;
}
int main()
{
	unsigned *o; long long *c, h;
	cudaMalloc(&o, 128); cudaMalloc(&c, 8);
	const char *names[] = { "match_any (identical values)", "match_any (32 distinct values)", "ballot", "shfl",
	    "smem atomicOr", "smem st+syncwarp+ld", "redux.add" };
	for (int m = 0; m < 7; m++) {
		k<<<1, 32>>>(o, c, m); cudaMemcpy(&h, c, 8, cudaMemcpyDeviceToHost);
		printf("%-34s %lld cycles per dependent op\n", names[m], h);
	}
	return 0;
}
