// dmma.cuh — the fp64 tensor-core MMA (DMMA) fragment op shared by als.cu and ease.cu.
// mma.sync m16n8k16 .f64 (PTX ISA): with g = lane / 4 and q = lane % 4,
//   a_i = A[g + 8 (i & 1)][q + 4 (i >> 1)]  (i < 8),   b_j = B[q + 4 j][g]  (j < 4),
//   c   = {(g, 2q), (g, 2q + 1), (g + 8, 2q), (g + 8, 2q + 1)}.
// Hopper has no fp64 wgmma; this is the fp64 tensor-core path.
#pragma once

namespace eb {

__device__ __forceinline__ void dmma(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
    asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
        "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
          "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

}  // namespace eb
