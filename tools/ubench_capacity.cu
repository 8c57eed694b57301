// Where is the L2 capacity cliff for a random read+2xRED table while 16 B/event stream through?
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
typedef uint64_t u64;
__device__ __forceinline__ u64 mix64(u64 z){ z=(z^(z>>30))*0xBF58476D1CE4E5B9ULL; z=(z^(z>>27))*0x94D049BB133111EBULL; return z^(z>>31);}
struct __align__(32) Slot { u64 a,b,c,d; };
template<int STREAM>
__global__ void k(Slot* t, u64 nslots, u64 n, u64* sink, const u64* keys, const u64* vals){
  u64 acc=0; u64 pol; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  for (u64 i=(u64)blockIdx.x*blockDim.x+threadIdx.x;i<n;i+=(u64)gridDim.x*blockDim.x){
    u64 key=i, val=i;
    if (STREAM){ asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;":"=l"(key):"l"(keys+i),"l"(pol)); asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;":"=l"(val):"l"(vals+i),"l"(pol)); key+=i; }
    u64 s = __umul64hi(mix64(key), nslots);
    Slot* p=t+s; u64 a,b,c,d;
    asm volatile("ld.global.relaxed.gpu.v2.u64 {%0,%1}, [%2];":"=l"(a),"=l"(b):"l"(p):"memory"); asm volatile("ld.global.relaxed.gpu.v2.u64 {%0,%1}, [%2];":"=l"(c),"=l"(d):"l"(&p->c):"memory"); acc+=a+b+c+d;
    asm volatile("red.global.relaxed.gpu.add.u64 [%0], %1;"::"l"(&p->d),"l"(1ULL):"memory");
    asm volatile("red.global.relaxed.gpu.max.s64 [%0], %1;"::"l"(&p->b),"l"((long long)val):"memory");
  }
  if (acc==0x1234567) *sink=acc;
}
int main(){
  u64 n = 1ull<<24; u64* sink; cudaMalloc(&sink,8);
  const int NB=6; u64 *keys[NB], *vals[NB];
  for(int i=0;i<NB;++i){ cudaMalloc(&keys[i], n*8); cudaMemset(keys[i],0,n*8); cudaMalloc(&vals[i], n*8); cudaMemset(vals[i],0,n*8);} 
  cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  int mbs[]={16,32,40,48,56,64,72,80,96,112,128,160,192};
  for (int mb: mbs){
    u64 slots=(u64)mb*1024*1024/32; Slot* t; cudaMalloc(&t, slots*32); cudaMemset(t,0,slots*32);
    for (int stream=0; stream<2; ++stream){
      // warm + 6 timed launches over distinct input buffers (like consecutive activations)
      float tot=0; 
      for (int rep=0; rep<NB+1; ++rep){
        cudaEventRecord(e0);
        if(stream) k<1><<<132*8,256>>>(t,slots,n,sink,keys[rep%NB],vals[rep%NB]); else k<0><<<132*8,256>>>(t,slots,n,sink,nullptr,nullptr);
        cudaEventRecord(e1); cudaEventSynchronize(e1); float ms; cudaEventElapsedTime(&ms,e0,e1); if(rep>0) tot+=ms;
      }
      printf("table %4d MB  %s  %.3f ms/launch  %.1f G ev/s\n", mb, stream?"+16B/ev stream (evict_first)":"no stream                   ", tot/NB, n/(tot/NB)/1e6);
    }
    cudaFree(t);
  }
  return 0;
}
