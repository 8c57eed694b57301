// Micro-benchmark: what do random 32-byte-sector reads and L2 reductions cost on this GPU?
// (informs the fold kernel's design)
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
typedef uint64_t u64;
__device__ __forceinline__ u64 mix64(u64 z){ z=(z^(z>>30))*0xBF58476D1CE4E5B9ULL; z=(z^(z>>27))*0x94D049BB133111EBULL; return z^(z>>31);}
struct __align__(32) Slot { u64 a,b,c,d; };
template<int MODE>
__global__ void k(Slot* t, u64 mask, u64 n, u64* sink, const u64* keys){
  u64 acc=0;
  for (u64 i=(u64)blockIdx.x*blockDim.x+threadIdx.x;i<n;i+=(u64)gridDim.x*blockDim.x){
    u64 key = keys ? keys[i] : i;
    u64 s = mix64(key) & mask;
    Slot* p=t+s;
    if (MODE==0 || MODE>=2){ u64 a,b,c,d; asm volatile("ld.global.relaxed.gpu.v2.u64 {%0,%1}, [%2];":"=l"(a),"=l"(b):"l"(p):"memory"); asm volatile("ld.global.relaxed.gpu.v2.u64 {%0,%1}, [%2];":"=l"(c),"=l"(d):"l"(&p->c):"memory"); acc+=a+b+c+d; }
    if (MODE==1 || MODE>=2){ asm volatile("red.global.relaxed.gpu.add.u64 [%0], %1;"::"l"(&p->d),"l"(1ULL):"memory"); }
    if (MODE==3){ asm volatile("red.global.relaxed.gpu.max.s64 [%0], %1;"::"l"(&p->b),"l"((long long)i):"memory"); }
    if (MODE==4){ asm volatile("red.global.relaxed.gpu.add.u32 [%0], %1;"::"l"((unsigned*)&p->d),"r"(1u):"memory"); }
    if (MODE==5){ atomicAdd((unsigned long long*)&p->d, 1ULL) ; }
  }
  if (acc==0x1234567) *sink=acc;
}
int main(){
  u64 n = 1ull<<26; u64* sink; cudaMalloc(&sink,8);
  u64* keys; cudaMalloc(&keys, n*8); cudaMemset(keys, 0, n*8);
  cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const char* names[]={"ld256","red.add.u64","ld256+red.add","ld256+red.add+red.max","ld256+red.add.u32(same sector)","ld256+atomicAdd(ret unused)"};
  for (int logs=15; logs<=23; logs+=2){
    u64 slots=1ull<<logs; Slot* t; cudaMalloc(&t, slots*32); cudaMemset(t,0,slots*32);
    for (int mode=0; mode<6; ++mode){
      for (int usekeys=0; usekeys<2; ++usekeys){
        float best=1e9;
        for (int rep=0; rep<3; ++rep){
          cudaEventRecord(e0);
          const u64* kp = usekeys? keys: nullptr;
          int grid=132*8;
          switch(mode){case 0:k<0><<<grid,256>>>(t,slots-1,n,sink,kp);break;case 1:k<1><<<grid,256>>>(t,slots-1,n,sink,kp);break;case 2:k<2><<<grid,256>>>(t,slots-1,n,sink,kp);break;case 3:k<3><<<grid,256>>>(t,slots-1,n,sink,kp);break;case 4:k<4><<<grid,256>>>(t,slots-1,n,sink,kp);break;default:k<5><<<grid,256>>>(t,slots-1,n,sink,kp);}
          cudaEventRecord(e1); cudaEventSynchronize(e1); float ms; cudaEventElapsedTime(&ms,e0,e1); if(ms<best)best=ms;
        }
        if (usekeys==0 || mode==2) printf("table %5llu KB  %-34s %s  %.3f ms  %.1f Gops/s\n",(unsigned long long)(slots*32/1024),names[mode],usekeys?"(+stream 8B/ev)":"               ",best,n/best/1e6);
      }
    }
    cudaFree(t);
  }
  // note: with usekeys all keys are 0 -> same slot; skip interpretation for that line (contention case)
  return 0;
}
