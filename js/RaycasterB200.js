// js/RaycasterB200.js -- Raycaster.intersectSplatMesh (src/raycaster/Raycaster.js:36-85) through the engine (not run here: no Node.js in
// the image).  The reference recurses over the SplatTree in JS and reads every splat of every reached leaf on the main thread; here the
// box tests, the per-splat tests and the sort by distance run on the GPU (gs_raycast) and only the nearest hits come back.
//
//   uploadSplatTreeForRaycast(engine, splatMesh.getSplatTree());        // once per tree: leaves + every node's box and parent
//   const hits = intersectSplatMeshB200(engine, raycaster, splatMesh);   // after raycaster.setFromCameraAndScreenPosition(...)
//
// The engine must be created with {rayRecords: 1}.  .ksplat / .ply / .splat scenes loaded through the engine get their ray records from
// the GPU decode; for arrays the caller packs, uploadRayRecords(engine, records, from, count, sceneTransformOrNull) takes 56-byte
// gs_ray_record rows (f64 centre[3], f32 scale[3], f32 rotation x y z w, u8 alpha, 3 pad bytes).
import * as THREE from 'three';
import { createRequire } from 'module';
const addon = createRequire(import.meta.url)('./build/Release/gsplat_b200.node');

// the reference's tree (one scene): leaves in nodesWithIndexes order, every node depth first with its parent
export function uploadSplatTreeForRaycast(engine, splatTree) {
    const subTree = splatTree.subTrees[0];
    const nodes = [], parents = [], leafNode = new Map();
    const visit = (node, parent) => {
        const me = nodes.length;
        nodes.push(node); parents.push(parent);
        leafNode.set(node, me);
        for (const child of node.children) visit(child, me);
    };
    visit(subTree.rootNode, -1);
    const leaves = subTree.nodesWithIndexes;
    const m = leaves.length, k = nodes.length;
    const center = new Float64Array(3 * m), lmin = new Float64Array(3 * m), lmax = new Float64Array(3 * m), offsets = new Uint32Array(m + 1);
    let total = 0;
    leaves.forEach((n) => { total += n.data.indexes.length; });
    const indexes = new Uint32Array(total);
    leaves.forEach((n, i) => {
        center.set([n.center.x, n.center.y, n.center.z], 3 * i); lmin.set([n.min.x, n.min.y, n.min.z], 3 * i); lmax.set([n.max.x, n.max.y, n.max.z], 3 * i);
        indexes.set(n.data.indexes, offsets[i]); offsets[i + 1] = offsets[i] + n.data.indexes.length;
    });
    addon.uploadSplatTree(engine, center, lmin, lmax, offsets, indexes, m);
    const nmin = new Float64Array(3 * k), nmax = new Float64Array(3 * k);
    nodes.forEach((n, i) => { nmin.set([n.min.x, n.min.y, n.min.z], 3 * i); nmax.set([n.max.x, n.max.y, n.max.z], 3 * i); });
    addon.uploadSplatTreeNodes(engine, nmin, nmax, Int32Array.from(parents), k, Uint32Array.from(leaves.map((n) => leafNode.get(n))), m);
}

// -> Hit-shaped objects {origin, normal, distance, splatIndex}, nearest first (all of them unless `capacity` is given)
export function intersectSplatMeshB200(engine, raycaster, splatMesh, outHits = [], capacity) {
    const fromLocal = new THREE.Matrix4().copy(splatMesh.matrixWorld);
    if (splatMesh.dynamicMode) fromLocal.multiply(splatMesh.getSceneTransform(0, new THREE.Matrix4()));
    const params = {
        origin: raycaster.ray.origin.toArray(), direction: raycaster.ray.direction.toArray(), fromLocal: fromLocal.elements,
        ellipsoid: raycaster.raycastAgainstTrueSplatEllipsoid ? 1 : 0, sceneVisible: splatMesh.getScene(0).visible ? 1 : 0,
    };
    let cap = capacity === undefined ? 64 : capacity;
    let out = new Float64Array(8 * Math.max(cap, 1));
    let total = addon.raycast(engine, params, out, cap);
    if (capacity === undefined && total > cap) {
        cap = total;
        out = new Float64Array(8 * cap);
        total = addon.raycast(engine, params, out, cap);
    }
    const idx = new Uint32Array(out.buffer);
    for (let i = 0; i < Math.min(cap, total); i++) {
        const b = 8 * i;
        outHits.push({
            origin: new THREE.Vector3(out[b], out[b + 1], out[b + 2]), normal: new THREE.Vector3(out[b + 3], out[b + 4], out[b + 5]),
            distance: out[b + 6], splatIndex: idx[2 * (b + 7)],
        });
    }
    return outHits;
}
